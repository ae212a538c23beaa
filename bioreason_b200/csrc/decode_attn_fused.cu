// Paged-KV decode attention for the GRPO rollout (replaces the HF generate() token loop + DynamicCache torch.cat growth,
// HF generation/utils.py:2760-2800; SURVEY.md §2.3 K8).
//
// KV cache layout (per layer): K and V are [n_pages, Hkv, 64, D] bf16 -- the 64 keys of one (page, kv head) are one
// contiguous 16 KB tile, i.e. exactly the shared-memory tile of the attention kernel.  A row's context is a page
// table; the G samples of a prompt group point at the SAME prompt pages (prefix sharing), so the shared-prefix pass treats
// the whole group as one problem (G x Hq/Hkv query vectors per kv head form the M dimension of the QK^T / PV mma tiles) and
// reads every prompt K/V tile once per group instead of G times.  Everything that changes from step to step (row lengths) is
// read from device memory, so one captured CUDA graph replays for every token.
//
// One launch per layer per decode step (the decode step is launch-latency sensitive): q/k RMSNorm + RoPE, KV append,
// prefix-shared + private paged attention and the split combine.
//
// Work items (blockIdx.x): first  n_groups*Hkv*SS  "shared" items  (group, kv head, split over the common prompt pages;
//                                 G x Hq/Hkv query vectors = the M dimension of the mma tiles),
//                          then   R*Hkv*SP         "private" items (row, kv head, split over the row's own pages).
// Every item ropes its own query vectors in shared memory (no roped copy of Q in HBM).  The private item whose page range
// contains the newest position also norm+ropes the new K, copies the new V and appends both to the row's page before
// loading it.  Partials (O, LSE) go to a workspace; the last item to arrive for a (row, kv head) pair merges them.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "attn_common.cuh"
using namespace attn;

namespace {

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16(x)); }
// two roundings with ONE conversion instruction (F2FP packs a pair; it issues at the special-function rate, so a prologue made of
// single-value roundings is bound by it)
__device__ __forceinline__ void rbf2(float& a, float& b) { const float2 r = br::unpack_bf16(br::pack_bf16(a, b)); a = r.x; b = r.y; }

struct FusedParams {
    const bf16* qkv; long long ld;        // raw (pre-norm, pre-rope) fused QKV of the new tokens [R, ld]
    const bf16 *qw, *kw;
    bf16 *kcache, *vcache;
    const int* page_table; int max_pages;
    const int* cur_len;
    int R, G, Hq, Hkv, GQ;
    int n_shared_pages, SS, SP, n_slots;
    float* part_o; float* part_lse; int* counters;      // [R,Hq,n_slots,D], [R,Hq,n_slots], [2][R*Hkv] (arrivals, finished pollers)
    bf16* out; long long ldo;
    float scale_log2, theta, eps;
    const float2* rope;                  // [n_pos, D/2] (cos, sin), bf16-rounded like HF's tables
    int rope_n_pos;
};

// cos/sin table: rope[pos, j] = (bf16(cos(pos * theta^(-2j/D))), bf16(sin(...))) -- the transcendental work of the decode loop, done once
__global__ void rope_table_kernel(float2* __restrict__ out, int n_pos, int half, float theta) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pos * half) return;
    const int pos = i / half, j = i % half;
    const float inv_freq = 1.0f / powf(theta, (float)(2 * j) / (float)(2 * half));
    float sn, cs;
    sincosf((float)pos * inv_freq, &sn, &cs);
    out[i] = make_float2(rbf(cs), rbf(sn));
}

// prefill: copy the (already roped) K and V of tokens [0, n_tok) of one prompt row into its pages
template <int D>
__global__ void kv_write_pages_kernel(const bf16* __restrict__ qkv, long long ld, int n_tok, int Hq, int Hkv, const int* __restrict__ pages,
                                      bf16* __restrict__ kcache, bf16* __restrict__ vcache) {
    const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wid >= n_tok * 2 * Hkv) return;
    const int tok = wid / (2 * Hkv), hh = wid % (2 * Hkv);
    const bool is_v = hh >= Hkv;
    const int kvh = is_v ? hh - Hkv : hh;
    const bf16* src = qkv + (long long)tok * ld + (long long)(Hq + hh) * D;
    const int page = pages[tok >> 6], slot = tok & 63;
    bf16* dst = (is_v ? vcache : kcache) + (((long long)page * Hkv + kvh) * 64 + slot) * D;
    for (int i = lane; i < D / 8; i += 32) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
}

// same arithmetic with the norm weights and the (cos, sin) pairs already in registers
template <int D>
__device__ __forceinline__ void norm_rope_words_pre(uint32_t wlo, uint32_t whi, const float (&wl)[D / 64], const float (&wh)[D / 64],
                                                    const float2 (&cs_sn)[D / 64], float eps, float (&olo)[D / 64], float (&ohi)[D / 64]) {
    constexpr int E = D / 64;
    const float2 a2 = br::unpack_bf16(wlo), b2 = br::unpack_bf16(whi);
    const float lo[E] = {a2.x, a2.y}, hi[E] = {b2.x, b2.y};
    const float ss = a2.x * a2.x + a2.y * a2.y + b2.x * b2.x + b2.y * b2.y;
    const float rstd = rsqrtf(br::warp_sum(ss) / (float)D + eps);
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const float a = rbf(wl[e] * rbf(lo[e] * rstd)), b = rbf(wh[e] * rbf(hi[e] * rstd));
        const float cs = cs_sn[e].x, sn = cs_sn[e].y;
        olo[e] = rbf(a * cs) + rbf(-b * sn);
        ohi[e] = rbf(b * cs) + rbf(a * sn);
    }
}

// Quarter-warp layout: 8 lanes own one 128-wide head vector (lane `sub` holds dims [8 sub, 8 sub + 8) of each half), so a warp ropes 4 query
// vectors at once; same arithmetic with the cos/sin pairs and the norm weights already in registers (all loads hoisted by the caller)
template <int D>
__device__ __forceinline__ void norm_rope_q8_pre(float (&lo)[8], float (&hi)[8], const float (&wl)[8], const float (&wh)[8], const float2 (&cs_sn)[8],
                                                 float eps) {
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) ss += lo[e] * lo[e] + hi[e] * hi[e];
    ss += __shfl_xor_sync(0xffffffffu, ss, 1); ss += __shfl_xor_sync(0xffffffffu, ss, 2); ss += __shfl_xor_sync(0xffffffffu, ss, 4);
    const float rstd = rsqrtf(ss / (float)D + eps);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        float a = lo[e] * rstd, b = hi[e] * rstd;
        rbf2(a, b);
        a *= wl[e]; b *= wh[e];
        rbf2(a, b);
        const float cs = cs_sn[e].x, sn = cs_sn[e].y;
        float ac = a * cs, bs = -b * sn, bc = b * cs, as = a * sn;
        rbf2(ac, bs); rbf2(bc, as);
        lo[e] = ac + bs;
        hi[e] = bc + as;
    }
}
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    const float2 a = br::unpack_bf16(v.x), b = br::unpack_bf16(v.y), c = br::unpack_bf16(v.z), d = br::unpack_bf16(v.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    return make_uint4(br::pack_bf16(f[0], f[1]), br::pack_bf16(f[2], f[3]), br::pack_bf16(f[4], f[5]), br::pack_bf16(f[6], f[7]));
}

// L2 loads of the two 32-bit words a lane owns of a 128-wide bf16 head vector (PDL chain: never through L1)
__device__ __forceinline__ void load_head_words(const bf16* src, int lane, uint32_t& wlo, uint32_t& whi) {
    wlo = __ldcg(reinterpret_cast<const unsigned int*>(src + lane * 2));
    whi = __ldcg(reinterpret_cast<const unsigned int*>(src + 64 + lane * 2));
}

// The two contractions of a tile run on mma.sync m16n8k16: the M dimension here is at most 32 query vectors, below the 64 rows of
// a Hopper warpgroup MMA.
template <int D>
__global__ void __launch_bounds__(64) decode_fused_kernel(const FusedParams p) {
    constexpr int BN = 64, TILE = 64 * D * 2, NT = 64, QROWS = 32, E = D / 64;
    extern __shared__ __align__(128) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;
    uint8_t* sQ = smem;                          // 32 x D
    uint8_t* sK = smem + QROWS * D * 2;
    uint8_t* sV = sK + 2 * TILE;
    auto qptr = [&](int s, int c) -> uint8_t* { return tile_ptr<D>(sQ, s, c); };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    br::launch_dependents();
    // ------------------------------------------------------------------------------------------------------------------
    // Everything up to grid_dep_wait() depends only on state the PREVIOUS kernel of the chain (this step's qkv GEMM) does not
    // touch: page table, cur_len, rope table, norm weights and the KV pages of earlier tokens.  It is issued before the wait,
    // so the KV fetch (DRAM latency, queued behind the weight stream) overlaps the qkv GEMM instead of following it.
    // ------------------------------------------------------------------------------------------------------------------
    const int n_groups = p.R / p.G;
    const int n_shared_items = (p.n_shared_pages > 0 && p.SS > 0) ? n_groups * p.Hkv * p.SS : 0;
    int item = blockIdx.x;
    const bool shared_pass = item < n_shared_items;
    int split, kvh, row_base, rows_per_unit, n_splits, slot_base;
    if (shared_pass) {
        split = item % p.SS; kvh = (item / p.SS) % p.Hkv; row_base = (item / (p.SS * p.Hkv)) * p.G;
        rows_per_unit = p.G; n_splits = p.SS; slot_base = 0;
    } else {
        item -= n_shared_items;
        split = item % p.SP; kvh = (item / p.SP) % p.Hkv; row_base = item / (p.SP * p.Hkv);
        rows_per_unit = 1; n_splits = p.SP; slot_base = n_shared_items ? p.SS : 0;
    }
    const int n_sh = n_shared_items ? p.n_shared_pages : 0;
    const int* table = p.page_table + (long long)row_base * p.max_pages;
    const long long page_stride = (long long)p.Hkv * 64 * D;

    int kv_len = 0, pg_lo, pg_hi;
    if (shared_pass) { pg_lo = split; pg_hi = n_sh; }
    else { kv_len = __ldcg(p.cur_len + row_base) + 1; pg_lo = n_sh + split; pg_hi = (kv_len + 63) >> 6; }
    // the page that receives this step's token (private pass): its tile may only be loaded after the append below
    const int newest_pg = shared_pass ? -1 : ((kv_len - 1) >> 6);
    const bool owns_newest = !shared_pass && newest_pg >= pg_lo && (newest_pg - pg_lo) % n_splits == 0;

    auto tile_src = [&](const bf16* cache, int pg) { return cache + (long long)table[pg] * page_stride + (long long)kvh * 64 * D; };
    auto issue_tile = [&](int st, int pg) {
            load_tile<D, NT>(sK + st * TILE, tile_src(p.kcache, pg), D, 0, 64, tid);
            load_tile<D, NT>(sV + st * TILE, tile_src(p.vcache, pg), D, 0, 64, tid);
    };
    const int pg1 = pg_lo + n_splits;
    const bool have0 = pg_lo < pg_hi, have1 = pg1 < pg_hi;
    const bool early0 = have0 && pg_lo != newest_pg, early1 = have1 && pg1 != newest_pg;
    if (early0) issue_tile(0, pg_lo);
    if (early1) issue_tile(1, pg1);
    cp_async_commit();

    // query-prep operands that do not depend on the new tokens: positions, norm weights, the rope pairs of the first pass.
    // NOTE on code size: this prologue runs once per CTA, so every instruction is a cold instruction-cache fetch; the 4 passes are a
    // real loop (one copy of the arithmetic, the next pass's rope pairs in flight) and there is no inline powf/sincosf fallback -- the
    // host always supplies the rope table (the fully unrolled version was ~10 k instructions and cost ~3 us of fetch stalls per launch).
    const int q4 = lane >> 3, sub = lane & 7;
    int posv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int s = warp * 16 + i * 4 + q4;
        const int rr = s / p.GQ;
        const bool ok = rr < rows_per_unit && (row_base + rr) < p.R;
        posv[i] = ok ? min(__ldcg(p.cur_len + row_base + rr), p.rope_n_pos - 1) : -1;
    }
    float wl[8], wh[8];
    { uint4 a = __ldg(reinterpret_cast<const uint4*>(p.qw + sub * 8)), b = __ldg(reinterpret_cast<const uint4*>(p.qw + 64 + sub * 8)); unpack8(a, wl); unpack8(b, wh); }
    // rope pairs of ALL four passes, requested here (before the dependency wait) and kept packed (the table holds bf16-rounded cos / sin,
    // so bf16x2 words lose nothing): a pass that fetched its pairs itself could not be shorter than an L2 round trip
    uint32_t tcp[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float4* tp = reinterpret_cast<const float4*>(p.rope + (long long)(posv[i] < 0 ? 0 : posv[i]) * (D / 2) + sub * 8);
#pragma unroll
        for (int e = 0; e < 4; ++e) { const float4 t4 = __ldg(tp + e); tcp[i][2 * e] = br::pack_bf16(t4.x, t4.y); tcp[i][2 * e + 1] = br::pack_bf16(t4.z, t4.w); }
    }
    // new-token K: norm weight + rope pair of the lane's two dims (owner item, warp 0)
    float2 kcs[E]; float kwl[E], kwh[E];
    if (owns_newest && warp == 0) {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int j = lane * E + e;
            kwl[e] = __bfloat162float(p.kw[j]); kwh[e] = __bfloat162float(p.kw[D / 2 + j]);
            kcs[e] = __ldg(p.rope + (long long)min(kv_len - 1, p.rope_n_pos - 1) * (D / 2) + j);
        }
    }
    br::grid_dep_wait();

    // ---- everything that depends on this step's qkv GEMM is requested at once: the raw query chunks and the new token's K / V
    {
        uint4 rl[4], rh[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int s = warp * 16 + i * 4 + q4;
            const int rr = s / p.GQ, hh = kvh * p.GQ + s % p.GQ;
            rl[i] = rh[i] = make_uint4(0, 0, 0, 0);
            if (posv[i] >= 0) {
                const bf16* src = p.qkv + (long long)(row_base + rr) * p.ld + (long long)hh * D;
                rl[i] = __ldcg(reinterpret_cast<const uint4*>(src + sub * 8));
                rh[i] = __ldcg(reinterpret_cast<const uint4*>(src + 64 + sub * 8));
            }
        }
        uint32_t kwlo = 0, kwhi = 0; uint4 vraw = make_uint4(0, 0, 0, 0);
        if (owns_newest) {
            if (warp == 0) load_head_words(p.qkv + (long long)row_base * p.ld + (long long)(p.Hq + kvh) * D, lane, kwlo, kwhi);
            else if (lane < D / 8) vraw = __ldcg(reinterpret_cast<const uint4*>(p.qkv + (long long)row_base * p.ld + (long long)(p.Hq + p.Hkv + kvh) * D) + lane);
        }
        // ---- queries: norm + rope (slot s -> row s / GQ, head kvh*GQ + s % GQ); 8 lanes per vector, 4 vectors per warp per pass, straight
        // from the registers the raw chunks landed in to their final (swizzled) place in the Q tile.  Slots are ordered by row: the passes
        // that hold a live query vector form a prefix (private items: ONE pass of warp 0, none of warp 1); dead slots get zeros.
        const int live_slots = min(rows_per_unit, max(p.R - row_base, 0)) * p.GQ - warp * 16;
        const int n_pass = live_slots <= 0 ? 0 : min(4, (live_slots + 3) >> 2);
        // A real loop (one copy of the arithmetic in the instruction cache: this code runs once per CTA, so straight-line code is bound by
        // instruction fetch); the pass's operands are picked out of the preloaded registers with selects instead of indexed arrays.
        auto pick4 = [](int i, const uint4& a, const uint4& b, const uint4& c, const uint4& d) {
            uint4 r;
            r.x = i == 0 ? a.x : (i == 1 ? b.x : (i == 2 ? c.x : d.x)); r.y = i == 0 ? a.y : (i == 1 ? b.y : (i == 2 ? c.y : d.y));
            r.z = i == 0 ? a.z : (i == 1 ? b.z : (i == 2 ? c.z : d.z)); r.w = i == 0 ? a.w : (i == 1 ? b.w : (i == 2 ? c.w : d.w));
            return r;
        };
#pragma unroll 1
        for (int i = 0; i < 4; ++i) {
            const int s = warp * 16 + i * 4 + q4;
            uint4 olo = make_uint4(0, 0, 0, 0), ohi = olo;
            if (i < n_pass) {                                          // warp-uniform
                const uint4 ql = pick4(i, rl[0], rl[1], rl[2], rl[3]), qh = pick4(i, rh[0], rh[1], rh[2], rh[3]);
                const int pos = i == 0 ? posv[0] : (i == 1 ? posv[1] : (i == 2 ? posv[2] : posv[3]));
                float lo[8], hi[8];
                float2 cs[8];
                unpack8(ql, lo); unpack8(qh, hi);
#pragma unroll
                for (int e = 0; e < 8; ++e) cs[e] = br::unpack_bf16(i == 0 ? tcp[0][e] : (i == 1 ? tcp[1][e] : (i == 2 ? tcp[2][e] : tcp[3][e])));
                norm_rope_q8_pre<D>(lo, hi, wl, wh, cs, p.eps);
                if (pos >= 0) { olo = pack8(lo); ohi = pack8(hi); }
            }
            *reinterpret_cast<uint4*>(qptr(s, sub)) = olo;
            *reinterpret_cast<uint4*>(qptr(s, 8 + sub)) = ohi;
        }
        // ---- append the new token's K / V (private item that owns the newest page)
        if (owns_newest) {
            const int pos = kv_len - 1;
            const int page = table[newest_pg], slot = pos & 63;
            if (warp == 0) {
                float olo[E], ohi[E];
                norm_rope_words_pre<D>(kwlo, kwhi, kwl, kwh, kcs, p.eps, olo, ohi);
                bf16* dst = p.kcache + ((long long)page * p.Hkv + kvh) * 64 * D + (long long)slot * D;
                const int j0 = lane * E;
                *reinterpret_cast<uint32_t*>(dst + j0) = br::pack_bf16(olo[0], olo[1]);
                *reinterpret_cast<uint32_t*>(dst + D / 2 + j0) = br::pack_bf16(ohi[0], ohi[1]);
            } else {
                bf16* dst = p.vcache + ((long long)page * p.Hkv + kvh) * 64 * D + (long long)slot * D;
                if (lane < D / 8) reinterpret_cast<uint4*>(dst)[lane] = vraw;
            }
            __threadfence();
        }
    }
    __syncthreads();
    // the newest page, if it is one of the first two tiles of this item, could not be fetched before the append
    if (have0 && !early0) issue_tile(0, pg_lo);
    if (have1 && !early1) issue_tile(1, pg1);
    cp_async_commit();

    const bool warp_live = shared_pass ? (warp * 16 < rows_per_unit * p.GQ) : (warp == 0);
    {
    uint32_t qf[D / 16][4];
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
        ldsm_x4(qf[kk], tile_ptr<D>(sQ, warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, kk * 2 + (lane >> 4)));
    cp_async_wait<0>();
    __syncthreads();

    float o[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    int it = 0;
    for (int pg = pg_lo; pg < pg_hi; pg += n_splits, ++it) {
        const int st = it & 1;
        uint8_t* cK = sK + st * TILE;
        uint8_t* cV = sV + st * TILE;
        if (it >= 1 && pg + n_splits < pg_hi) issue_tile(st ^ 1, pg + n_splits);      // tiles 0 and 1 were issued before the loop
        cp_async_commit();
        if (warp_live) {
            float s[BN / 8][4];
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
            for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
                for (int np = 0; np < BN / 16; ++np) {
                    uint32_t kf[4];
                    ldsm_x4(kf, tile_ptr<D>(cK, np * 16 + (lane & 7) + (lane >> 4) * 8, kk * 2 + ((lane >> 3) & 1)));
                    mma16816(s[2 * np], qf[kk], kf[0], kf[1]);
                    mma16816(s[2 * np + 1], qf[kk], kf[2], kf[3]);
                }
            }
            const int nbase = pg * BN;
            const bool need_mask = !shared_pass && (nbase + BN > kv_len);
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < BN / 8; ++nt) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float v = s[nt][e] * p.scale_log2;
                    if (need_mask) { const int j = nbase + nt * 8 + 2 * t + (e & 1); v = (j < kv_len) ? v : -INFINITY; }
                    s[nt][e] = v;
                }
                mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
                mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
            const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
            const float a0 = exp2f(m0 - ms0), a1 = exp2f(m1 - ms1);
            m0 = mn0; m1 = mn1;
            float rs0 = 0.f, rs1 = 0.f;
            uint32_t pf[BN / 16][4];
#pragma unroll
            for (int nt = 0; nt < BN / 8; ++nt) {
                const float p0 = exp2f(s[nt][0] - ms0), p1 = exp2f(s[nt][1] - ms0);
                const float p2 = exp2f(s[nt][2] - ms1), p3 = exp2f(s[nt][3] - ms1);
                rs0 += p0 + p1; rs1 += p2 + p3;
                pf[nt >> 1][(nt & 1) * 2 + 0] = br::pack_bf16(p0, p1);
                pf[nt >> 1][(nt & 1) * 2 + 1] = br::pack_bf16(p2, p3);
            }
            l0 = l0 * a0 + rs0; l1 = l1 * a1 + rs1;
#pragma unroll
            for (int i = 0; i < D / 8; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
#pragma unroll
            for (int kk = 0; kk < BN / 16; ++kk) {
#pragma unroll
                for (int dp = 0; dp < D / 16; ++dp) {
                    uint32_t vf[4];
                    ldsm_x4_t(vf, tile_ptr<D>(cV, kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dp * 2 + (lane >> 4)));
                    mma16816(o[2 * dp], pf[kk], vf[0], vf[1]);
                    mma16816(o[2 * dp + 1], pf[kk], vf[2], vf[3]);
                }
            }
        }
        cp_async_wait<0>();
        __syncthreads();
    }

    // ---- partials
    if (warp_live) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float LN2 = 0.6931471805599453f;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int s_idx = warp * 16 + g + half * 8;
            const int rr = s_idx / p.GQ, hh = kvh * p.GQ + s_idx % p.GQ;
            if (rr >= rows_per_unit || row_base + rr >= p.R) continue;
            const float l = half ? l1 : l0, m = half ? m1 : m0;
            const float inv = l > 0.f ? 1.f / l : 0.f;
            const long long base = ((long long)(row_base + rr) * p.Hq + hh) * p.n_slots + slot_base + split;
            float* po = p.part_o + base * D;
#pragma unroll
            for (int dt = 0; dt < D / 8; ++dt) {
                const float x = half ? o[dt][2] : o[dt][0], y = half ? o[dt][3] : o[dt][1];
                __stcg(reinterpret_cast<float2*>(po + dt * 8 + 2 * t), make_float2(x * inv, y * inv));
            }
            if (t == 0) __stcg(p.part_lse + base, l > 0.f ? m * LN2 + logf(l) : -INFINITY);
        }
    }
    }
    // ---- arrival counters: one per (row, kv head).  Every item publishes its partial and arrives; the SP private items of a
    //      (row, kv head) pair then ALL merge -- each a contiguous share of the pair's GQ x D output -- so the 64 merges of a step run on
    //      64 x SP CTAs and every thread has its whole gather (<= 32 slots of one float4 column) in flight in one L2 round trip.
    //      (A single merger per pair needed three dependent rounds of loads: it was the tail of the launch, ~4 us after the last
    //      arrival.)  All items of a launch are co-resident (checked on the host), so the bounded spin cannot deadlock.
    //      A row's GQ query vectors live in ONE warp (16 % GQ == 0), so a warp publishes its rows by itself: stores, __syncwarp, one
    //      release-reduction per row -- no CTA barrier, no fence, no returning atomic on the way out.
    __syncwarp();
    if (warp_live) {
        const int rows_in_warp = 16 / p.GQ;                         // a warp holds 16 / GQ rows
        const int rr = shared_pass ? warp * rows_in_warp + lane : 0;
        if (lane < (shared_pass ? rows_in_warp : 1) && rr < rows_per_unit && row_base + rr < p.R)
            asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(p.counters + (row_base + rr) * p.Hkv + kvh) : "memory");
    }
    if (shared_pass) return;
    if (tid == 0) {
        int* c = p.counters + row_base * p.Hkv + kvh;
        int seen;
        do { asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(c) : "memory"); } while (seen < p.n_slots);
        // the last of the SP pollers to get here resets both words for the next launch (nobody arrives or polls after that)
        int* dn = p.counters + p.R * p.Hkv + row_base * p.Hkv + kvh;
        if (atomicAdd(dn, 1) == p.SP - 1) { *c = 0; *dn = 0; }
    }
    __syncthreads();
    {
        // Every thread owns one float4 column of one head: it loads the head's slot LSEs itself (the same addresses across the threads
        // of a head: broadcast) together with its column of every slot -- ONE L2 round trip -- and derives the slot weights redundantly
        // in a fixed order (n_slots <= 32 exponentials per thread are cheaper than a second dependent trip through shared memory).
        const int row = row_base;
        const int per_row = p.GQ * (D / 4);                            // float4 chunks of this (row, kv head) output
        const int lo = (per_row * split) / p.SP, hi = (per_row * (split + 1)) / p.SP;
        for (int idx = lo + tid; idx < hi; idx += NT) {
            const int hl = idx / (D / 4), d0 = (idx % (D / 4)) * 4;
            const long long hb = ((long long)row * p.Hq + kvh * p.GQ + hl) * p.n_slots;
            const float* po = p.part_o + hb * D + d0;
            float ls[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) ls[j] = j < p.n_slots ? __ldcg(p.part_lse + hb + j) : -INFINITY;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float mx = -INFINITY, den = 0.f;
            bool have_w = false;
#pragma unroll 1
            for (int s0 = 0; s0 < p.n_slots; s0 += 24) {
                float4 va[24];
#pragma unroll
                for (int j = 0; j < 24; ++j)
                    va[j] = (s0 + j < p.n_slots) ? __ldcg(reinterpret_cast<const float4*>(po + (long long)(s0 + j) * D)) : make_float4(0.f, 0.f, 0.f, 0.f);
                if (!have_w) {                                         // slot weights: softmax over the slots' LSEs, fixed order
#pragma unroll
                    for (int j = 0; j < 32; ++j) mx = fmaxf(mx, ls[j]);
#pragma unroll
                    for (int j = 0; j < 32; ++j) { ls[j] = (ls[j] == -INFINITY) ? 0.f : __expf(ls[j] - mx); den += ls[j]; }
                    den = den > 0.f ? 1.f / den : 0.f;
                    have_w = true;
                }
#pragma unroll
                for (int j = 0; j < 24; ++j) {                         // fixed slot order: deterministic
                    const float w = (s0 == 0 ? ls[j] : ls[(24 + j) & 31]) * den;     // second batch: slots 24..31
                    if (s0 + j < p.n_slots) { acc.x += w * va[j].x; acc.y += w * va[j].y; acc.z += w * va[j].z; acc.w += w * va[j].w; }
                }
            }
            *reinterpret_cast<uint2*>(p.out + (long long)row * p.ldo + (long long)(kvh * p.GQ + hl) * D + d0) =
                make_uint2(br::pack_bf16(acc.x, acc.y), br::pack_bf16(acc.z, acc.w));
        }
    }
}

}  // namespace

extern "C" {

int br_kv_write_pages(const void* qkv, int64_t ld, int n_tok, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* pages, void* kcache,
                      void* vcache, void* stream) {
    BR_CHECK_ARG(head_dim == 128 && n_tok > 0, "kv_write_pages: head_dim 128, n_tok > 0");
    const int warps = n_tok * 2 * n_kv_heads, wpb = 8;
    kv_write_pages_kernel<128><<<(warps + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>((const bf16*)qkv, ld, n_tok, n_q_heads, n_kv_heads,
                                                                                             pages, (bf16*)kcache, (bf16*)vcache);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int64_t br_decode_fused_workspace_bytes(int R, int n_q_heads, int n_kv_heads, int head_dim, int n_slots) {
    return (int64_t)R * n_q_heads * n_slots * (head_dim + 1) * sizeof(float) + 2 * (int64_t)R * n_kv_heads * sizeof(int);
}

int br_rope_table(float* out, int n_pos, int head_dim, float theta, void* stream) {
    BR_CHECK_ARG(n_pos > 0 && head_dim % 2 == 0, "rope_table: bad shape");
    const int n = n_pos * (head_dim / 2);
    rope_table_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>((float2*)out, n_pos, head_dim / 2, theta);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_decode_attn_fused(const void* qkv_raw, int64_t ld, const void* q_norm_w, const void* k_norm_w, void* kcache, void* vcache,
                         const int32_t* page_table, int max_pages, const int32_t* cur_len, int R, int G, int n_q_heads, int n_kv_heads,
                         int head_dim, int n_shared_pages, int splits_shared, int splits_private, float scale, float theta, float eps,
                         const float* rope_table, int rope_n_pos, void* workspace, void* out, int64_t ldo, void* stream) {
    BR_CHECK_ARG(head_dim == 128, "decode_attn_fused: head_dim 128 only");
    BR_CHECK_ARG(R > 0 && G > 0 && R % G == 0 && G <= 64, "decode_attn_fused: R=%d must be a multiple of G=%d (<= 64)", R, G);
    const int GQ = n_q_heads / n_kv_heads;
    BR_CHECK_ARG(GQ <= 16 && 16 % GQ == 0 && G * GQ <= 32, "decode_attn_fused: G * Hq/Hkv = %d query vectors per kv head exceed 32", G * GQ);
    BR_CHECK_ARG(splits_private >= 1 && splits_shared >= 0 && splits_private + splits_shared <= 32 && q_norm_w && k_norm_w, "decode_attn_fused: bad arguments (<= 32 splits)");
    BR_CHECK_ARG(rope_table && rope_n_pos > 0, "decode_attn_fused: the cos/sin table of br_rope_table (covering every position of the rollout) is required");
    constexpr int D = 128;
    FusedParams p;
    p.qkv = (const bf16*)qkv_raw; p.ld = ld; p.qw = (const bf16*)q_norm_w; p.kw = (const bf16*)k_norm_w;
    p.kcache = (bf16*)kcache; p.vcache = (bf16*)vcache; p.page_table = page_table; p.max_pages = max_pages; p.cur_len = cur_len;
    p.R = R; p.G = G; p.Hq = n_q_heads; p.Hkv = n_kv_heads; p.GQ = GQ;
    const int use_shared = (n_shared_pages > 0 && splits_shared > 0) ? 1 : 0;
    p.n_shared_pages = use_shared ? n_shared_pages : 0; p.SS = use_shared ? splits_shared : 0; p.SP = splits_private;
    p.n_slots = p.SS + p.SP;
    p.part_o = (float*)workspace;
    p.part_lse = p.part_o + (int64_t)R * n_q_heads * p.n_slots * D;
    p.counters = (int*)(p.part_lse + (int64_t)R * n_q_heads * p.n_slots);
    p.out = (bf16*)out; p.ldo = ldo; p.scale_log2 = scale * 1.4426950408889634f; p.theta = theta; p.eps = eps;
    p.rope = (const float2*)rope_table; p.rope_n_pos = rope_table ? rope_n_pos : 0;
    constexpr int SMEM = 32 * D * 2 + 4 * 64 * D * 2;
    static bool done = false;
    if (!done) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(decode_fused_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        done = true;
    }
    const int items = (use_shared ? (R / G) * n_kv_heads * p.SS : 0) + R * n_kv_heads * p.SP;
    const int per_sm = 3;
    BR_CHECK_ARG(items <= per_sm * br_num_sms(), "decode_attn_fused: %d work items exceed the co-resident capacity (%d per SM) the in-kernel merge relies on", items, per_sm);
    BR_CHECK_CUDA(br_launch_pdl(decode_fused_kernel<D>, dim3(items), dim3(64), (size_t)SMEM, (cudaStream_t)stream, p));
    return BR_OK;
}

}  // extern "C"
