// Full-vocabulary rollout sampler (br_sample_next_full): temperature -> top-k (0: off, no cap on the kept set) -> top-p -> min-p ->
// inverse-CDF draw, for any top_k >= 0.  sampler.cu keeps at most 1024 candidates per row; here top_p = 0.95 on a nearly flat row keeps
// ~10^5 tokens, so every cut is a threshold over the whole row, found by exact radix select on multi-CTA passes.
//
// Contract (z' = z after the repetition penalty and the min_new_tokens EOS mask when processors are on, else z):
//   top-k     top_k = 0: off (every finite value kept).  top_k >= 1 is clamped to V; every value >= the k-th is kept, ties included.
//   top-p     the kept tokens ordered by value desc, id asc; drop from the end while the cumulative probability at T is <= 1 - p; the
//             first always stays.  Among equal values the higher ids are dropped first.
//   min-p     after top-p: drop e_j = exp((z'_j - z'_max) / T) < min_p (the maximum stays: e = 1).
//   draw      inverse CDF over the kept tokens in ascending id with uniforms[step * R + r]; a token at -inf is never drawn.
//   logp      z[y] - logsumexp(z) over the raw row at T = 1, from the chunk statistics of the two-stage sampler (bit-equal to
//             br_sample_next_2stage_logp's for the same token).
//   A row with no finite processed value draws pad_id (its logp is the raw row's at pad_id).  Finished rows emit pad.
//
// Arithmetic.  M = the row's maximum z' (the chunk maxima, combined by fmaxf: exact).  Every pass computes a token's weight with the
// same instructions, e = exp(fp64((z' - M) / T)) in fp64, and its 64-bit fixed-point mass q = rint(e 2^40)
// (e <= 1 and V < 2^23, so every row sum fits in 63 bits).  Integer sums are exact in any order, so the histograms are reduced with
// integer atomics and the result does not depend on scheduling; there is no floating-point atomic.
//   top-k: 3 radix passes (11 / 11 / 10 key bits) over counts find the k-th value exactly.
//   top-p: need = ceil(p Q) with Q the kept mass (exact, 128-bit); keep the shortest prefix in (value desc, id asc) order whose mass
//          reaches need (equivalent to dropping while the suffix is <= (1 - p) Q): 3 radix passes over masses find its last value v*,
//          and the number of ties of v* to keep is ceil(rest / q(v*)), the lowest ids.
//   draw:  target = floor(u K) (128-bit), K the kept mass; the chunk from the per-chunk kept masses, then a block scan of that chunk
//          in id order: the first token whose running mass exceeds target.
// Every pass is one grid of (chunks, R) CTAs over 4096-logit chunks; the last CTA of a row (integer arrival counter) makes the row's
// selection.  The first kernel zeroes the row's histograms and counters, and each pass's last CTA re-zeroes the histogram it read, so
// a captured call needs no host-side reset.  The launch sequence depends only on the arguments (top_k, top_p), never on the data.
#include "sampler_common.cuh"
#include "../../include/bioreason_b200.h"

namespace {

constexpr int FCHUNK = 4096, FTHREADS = 256, FPER = FCHUNK / FTHREADS, FBINS2 = 2048, NARRIVE = 8;
constexpr double QSCALE = 1099511627776.0;                    // 2^40

struct RowSel {
    uint32_t kkey;               // top-k: keep key >= kkey (0: every finite value)
    uint32_t cut_key;            // the final cut value: keep key > cut_key, and the first ntie ties of it in id order
    int ntie;
    uint32_t prefix;             // radix select in progress
    int rem_cnt;
    int empty;                   // no finite processed value
    unsigned long long rem_mass;
};

struct FullWs {
    RowSel* sel;                 // [R]
    int* arrive;                 // [R, NARRIVE]
    float* cmax;                 // [R, n_chunks]  chunk maxima of z'
    float2* stats;               // [R, n_chunks]  raw (m_c, s_c) of the log-prob
    unsigned long long* cmass;   // [R, n_chunks]  draw: mass strictly above the cut
    int* ctie;                   // [R, n_chunks]  draw: ties of the cut
    int* hcnt;                   // [R, 2048]
    unsigned long long* hmass;   // [R, 2048]
};

struct FullArgs {
    const float* logits; long long ld; int V; int n_chunks;
    float temperature; int top_k; float top_p;
    Proc pr;
};

__device__ __forceinline__ float key_to_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// the one instruction sequence every pass uses for a token's weight and fixed-point mass.  fp64: an fp32 exp's relative error, summed
// over 10^5 kept tokens, is as large as a typical token's weight on a nearly flat row; in fp64 the fixed-point rounding dominates.
__device__ __forceinline__ double weight(float z, float M, float T) { return exp(__ddiv_rn((double)z - (double)M, (double)T)); }
__device__ __forceinline__ unsigned long long fixmass(double e) { return __double2ull_rn(e * QSCALE); }

// floor or ceil of f * Q for fp32 f in [0, 1) and Q < 2^63, exactly
__device__ __forceinline__ unsigned long long scale_exact(float f, unsigned long long Q, bool ceil_) {
    const uint32_t b = __float_as_uint(f);
    const int ex = (b >> 23) & 255;
    const uint32_t man = (b & 0x7fffffu) | (ex ? 0x800000u : 0u);
    const int shift = ex ? 150 - ex : 149;                     // f = man 2^-shift
    const unsigned __int128 prod = (unsigned __int128)man * Q;
    if (prod == 0) return 0;
    if (shift >= 128) return ceil_ ? 1ull : 0ull;
    const unsigned __int128 r = ceil_ ? (prod + (((unsigned __int128)1 << shift) - 1)) >> shift : prod >> shift;
    return (unsigned long long)r;
}

// the row's z' values of this chunk, 16 per thread at base + i * 256 + tid (-inf past V)
template <bool PROC>
__device__ __forceinline__ void load_chunk(const FullArgs& a, int row, int base, float (&v)[FPER]) {
    const float* x = a.logits + (long long)row * a.ld;
    const int tid = threadIdx.x;
#pragma unroll
    for (int i = 0; i < FPER; ++i) {
        const int idx = base + i * FTHREADS + tid;
        v[i] = idx < a.V ? __ldcg(x + idx) : -INFINITY;
    }
    if constexpr (PROC) {
        const int step = a.pr.step ? __ldcg(a.pr.step) : 0;
        const bool block_eos = a.pr.eos >= 0 && step < a.pr.min_new;
        const uint32_t* pres = a.pr.presence ? a.pr.presence + (long long)row * ((a.V + 31) >> 5) : nullptr;
#pragma unroll
        for (int i = 0; i < FPER; ++i) {
            const int idx = base + i * FTHREADS + tid;
            if (idx < a.V) v[i] = proc_logit(v[i], proc_in_set(pres, idx), block_eos && idx == a.pr.eos, a.pr.theta);
        }
    }
}
template <bool PROC>
__device__ __forceinline__ float proc_one(const FullArgs& a, int row, int idx, bool block_eos) {
    float z = __ldcg(a.logits + (long long)row * a.ld + idx);
    if constexpr (PROC) {
        const uint32_t* pres = a.pr.presence ? a.pr.presence + (long long)row * ((a.V + 31) >> 5) : nullptr;
        z = proc_logit(z, proc_in_set(pres, idx), block_eos && idx == a.pr.eos, a.pr.theta);
    }
    return z;
}

__device__ __forceinline__ float row_max(const FullWs& w, const FullArgs& a, int row, float* s_red) {
    float m = -INFINITY;
    for (int c = threadIdx.x; c < a.n_chunks; c += FTHREADS) m = fmaxf(m, __ldcg(w.cmax + (long long)row * a.n_chunks + c));
    return block_max(m, s_red);
}

// "last CTA of the row": every CTA calls this after its global atomics / writes; true in the CTA that arrives last
__device__ __forceinline__ bool arrive_last(int* counter, int n, int* s_flag) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) *s_flag = atomicAdd(counter, 1) == n - 1;
    __syncthreads();
    const bool last = *s_flag;
    if (last) __threadfence();
    return last;
}

template <typename T>
__device__ __forceinline__ T warp_incl_scan(T v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    return v;
}
// exclusive block scan over FTHREADS threads; *total gets the sum; s: 8 + 1 elements
template <typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* s, T* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const T incl = warp_incl_scan(v);
    if (lane == 31) s[warp] = incl;
    __syncthreads();
    T before = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < FTHREADS / 32; ++w) { const T c = s[w]; tot += c; if (w < warp) before += c; }
    __syncthreads();
    *total = tot;
    return before + incl - v;
}

// warp 0: bin b (descending) with sum(bins > b) < rem <= sum(bins >= b); returns b, rem -= sum(bins > b)
template <typename T>
__device__ int select_desc(const T* hist, int nb, T& rem, int* s_b, T* s_rem) {
    const int lane = threadIdx.x & 31;
    const int per = nb / 32;
    const int hi = nb - 1 - lane * per;
    T sum = 0;
    for (int i = 0; i < per; ++i) sum += __ldcg(hist + hi - i);
    const T incl = warp_incl_scan(sum);
    const T excl = incl - sum;
    if (excl < rem && incl >= rem) {
        T acc = excl; int b = hi;
        for (int i = 0; i < per; ++i) {
            b = hi - i;
            const T h = __ldcg(hist + b);
            if (acc + h >= rem) break;
            acc += h;
        }
        *s_b = b; *s_rem = rem - acc;
    }
    __syncwarp();
    rem = *s_rem;
    return *s_b;
}

// ---- kernel 1: chunk maxima of z', the log-prob's raw chunk statistics, and the row's selection state reset
template <bool LOGP, bool PROC>
__global__ void __launch_bounds__(FTHREADS) full_stats_kernel(FullArgs a, FullWs w) {
    __shared__ float s_red[32];
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    br::launch_dependents();
    br::grid_dep_wait();
    const int base = chunk * FCHUNK;
    float v[FPER];
    if constexpr (LOGP) {
        // the raw chunk statistics, with the arithmetic of the two-stage sampler's stage 1
        const float* x = a.logits + (long long)row * a.ld;
#pragma unroll
        for (int i = 0; i < FPER; ++i) { const int idx = base + i * FTHREADS + tid; v[i] = idx < a.V ? __ldcg(x + idx) : -INFINITY; }
        float mr = -INFINITY;
#pragma unroll
        for (int i = 0; i < FPER; ++i) mr = fmaxf(mr, v[i]);
        mr = block_max(mr, s_red);
        float s = 0.f;
        if (mr > -INFINITY) {
#pragma unroll
            for (int i = 0; i < FPER; ++i) s += expf(v[i] - mr);
        }
        s = block_sum(s, s_red);
        if (tid == 0) w.stats[(long long)row * a.n_chunks + chunk] = make_float2(mr, s);
    }
    load_chunk<PROC>(a, row, base, v);
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < FPER; ++i) mx = fmaxf(mx, v[i]);
    mx = block_max(mx, s_red);
    if (tid == 0) w.cmax[(long long)row * a.n_chunks + chunk] = mx;
    for (int i = chunk * FTHREADS + tid; i < FBINS2; i += a.n_chunks * FTHREADS) {
        w.hcnt[(long long)row * FBINS2 + i] = 0;
        w.hmass[(long long)row * FBINS2 + i] = 0ull;
    }
    if (chunk == 0) {
        if (tid < NARRIVE) w.arrive[row * NARRIVE + tid] = 0;
        if (tid == 0) w.sel[row] = RowSel{0u, 0u, 0x7fffffff, 0u, 0, 0, 0ull};
    }
}

// ---- kernels 2..7: one radix pass of a cut.  MASS = false: top-k (counts), true: top-p (fixed-point masses over the top-k set)
template <bool PROC, bool MASS>
__global__ void __launch_bounds__(FTHREADS) full_select_kernel(FullArgs a, FullWs w, int pass, int arrive_slot) {
    __shared__ int s_cnt[FBINS2];
    __shared__ unsigned long long s_mass[MASS ? FBINS2 : 1];
    __shared__ float s_red[32];
    __shared__ int s_flag, s_b;
    __shared__ unsigned long long s_rem;
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    br::launch_dependents();
    br::grid_dep_wait();
    RowSel* st = w.sel + row;
    const uint32_t kkey = __ldcg(&st->kkey), prefix = __ldcg(&st->prefix);
    const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
    const int nb = pass == 2 ? 1024 : 2048;
    float v[FPER];
    load_chunk<PROC>(a, row, chunk * FCHUNK, v);
    float M = 0.f;
    if constexpr (MASS) M = row_max(w, a, row, s_red);
    const float T = a.temperature;
    for (int i = tid; i < nb; i += FTHREADS) { s_cnt[i] = 0; if constexpr (MASS) s_mass[i] = 0ull; }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < FPER; ++i) {
        const uint32_t key = fkey(v[i]);
        bool in = v[i] > -INFINITY && key >= kkey;
        if (pass == 1) in &= (key >> 21) == prefix; else if (pass == 2) in &= (key >> 10) == prefix;
        if (in) {
            const int b = (key >> shift) & (nb - 1);
            atomicAdd(&s_cnt[b], 1);
            if constexpr (MASS) atomicAdd(&s_mass[b], fixmass(weight(v[i], M, T)));
        }
    }
    __syncthreads();
    int* hc = w.hcnt + (long long)row * FBINS2;
    unsigned long long* hm = w.hmass + (long long)row * FBINS2;
    for (int i = tid; i < nb; i += FTHREADS) {
        if (s_cnt[i]) { atomicAdd(hc + i, s_cnt[i]); if constexpr (MASS) atomicAdd(hm + i, s_mass[i]); }
    }
    if (!arrive_last(w.arrive + row * NARRIVE + arrive_slot, a.n_chunks, &s_flag)) return;
    // ---- the row's selection (last CTA)
    if (tid < 32 && !__ldcg(&st->empty)) {
        if (!MASS) {
            int rem = pass == 0 ? 0 : __ldcg(&st->rem_cnt);
            if (pass == 0) {
                int n_fin = 0;
                for (int i = tid; i < nb; i += 32) n_fin += __ldcg(hc + i);
                for (int o = 16; o > 0; o >>= 1) n_fin += __shfl_xor_sync(0xffffffffu, n_fin, o);
                rem = min(a.top_k, n_fin);                         // fewer finite values than k: the k-th is -inf, keep them all
            }
            if (rem == 0) {
                if (tid == 0) st->empty = 1;
            } else {
                __shared__ int s_remi;
                const int b = select_desc<int>(hc, nb, rem, &s_b, &s_remi);
                if (tid == 0) {
                    const uint32_t p = pass == 0 ? (uint32_t)b : ((prefix << (pass == 1 ? 11 : 10)) | (uint32_t)b);
                    st->prefix = p; st->rem_cnt = rem;
                    if (pass == 2) { st->kkey = p; st->cut_key = p; st->ntie = 0x7fffffff; }
                }
            }
        } else {
            unsigned long long rem = pass == 0 ? 0ull : __ldcg(&st->rem_mass);
            if (pass == 0) {
                unsigned long long tot = 0ull;
                for (int i = tid; i < nb; i += 32) tot += __ldcg(hm + i);
                for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
                rem = scale_exact(a.top_p, tot, true);             // need = ceil(p Q) >= 1 (Q >= 2^40: the maximum has e = 1)
            }
            if (rem == 0ull) {
                if (tid == 0) st->empty = 1;
            } else {
                const int b = select_desc<unsigned long long>(hm, nb, rem, &s_b, &s_rem);
                if (tid == 0) {
                    const uint32_t p = pass == 0 ? (uint32_t)b : ((prefix << (pass == 1 ? 11 : 10)) | (uint32_t)b);
                    st->prefix = p; st->rem_mass = rem;
                    if (pass == 2) {
                        // every tie of v* has the same mass q*; keep the lowest-id ceil(rem / q*) of them
                        const unsigned long long q = __ldcg(hm + b) / (unsigned long long)__ldcg(hc + b);
                        st->cut_key = p; st->ntie = (int)((rem + q - 1) / q);
                    }
                }
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < nb; i += FTHREADS) { hc[i] = 0; if constexpr (MASS) hm[i] = 0ull; }   // zero for the next pass
}

// ---- last kernel: per-chunk kept masses, then (last CTA of the row) the draw, the log-prob and the bookkeeping
template <bool LOGP, bool PROC>
__global__ void __launch_bounds__(FTHREADS) full_draw_kernel(FullArgs a, FullWs w, int arrive_slot, const float* __restrict__ uniforms,
                                                             const int* __restrict__ step_ptr, int R, int max_steps, long long eos_id,
                                                             long long pad_id, int* __restrict__ finished, long long* __restrict__ tokens,
                                                             long long* __restrict__ next_ids, float* __restrict__ logp) {
    __shared__ float s_red[32];
    __shared__ unsigned long long s_u64[FTHREADS / 32];
    __shared__ int s_i32[FTHREADS / 32];
    __shared__ int s_flag, s_choice, s_chunk, s_tb;
    __shared__ unsigned long long s_before, s_target;
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    br::launch_dependents();
    br::grid_dep_wait();
    const RowSel* st = w.sel + row;
    const uint32_t cut = __ldcg(&st->cut_key);
    const int ntie = __ldcg(&st->ntie);
    const float M = row_max(w, a, row, s_red);
    const float T = a.temperature;
    const double min_p = PROC ? (double)a.pr.min_p : 0.0;
    const int step = step_ptr ? __ldcg(step_ptr) : 0;
    auto kept = [&](float z, double e) { return z > -INFINITY && fkey(z) >= cut && !(min_p > 0.0 && e < min_p); };
    {
        float v[FPER];
        load_chunk<PROC>(a, row, chunk * FCHUNK, v);
        unsigned long long m = 0ull; int t = 0;
#pragma unroll
        for (int i = 0; i < FPER; ++i) {
            const double e = weight(v[i], M, T);
            if (kept(v[i], e)) { if (fkey(v[i]) == cut) ++t; else m += fixmass(e); }
        }
        unsigned long long msum; int tsum;
        block_excl_scan<unsigned long long>(m, s_u64, &msum);
        block_excl_scan<int>(t, s_i32, &tsum);
        if (tid == 0) { w.cmass[(long long)row * a.n_chunks + chunk] = msum; w.ctie[(long long)row * a.n_chunks + chunk] = tsum; }
    }
    if (!arrive_last(w.arrive + row * NARRIVE + arrive_slot, a.n_chunks, &s_flag)) return;
    // ---- the draw (last CTA of the row)
    const float qz = key_to_float(cut);
    const unsigned long long qcut = fixmass(weight(qz, M, T));
    const bool empty = __ldcg(&st->empty) || !(M > -INFINITY);
    if (tid == 0) {
        s_chunk = -1;
        if (!empty) {
            unsigned long long K = 0ull;
            int tb = 0;
            for (int c = 0; c < a.n_chunks; ++c) {
                const int t = __ldcg(w.ctie + (long long)row * a.n_chunks + c);
                const int kt = min(t, max(0, ntie - tb)); tb += t;
                K += __ldcg(w.cmass + (long long)row * a.n_chunks + c) + (unsigned long long)kt * qcut;
            }
            const float u = uniforms[(long long)step * R + row];
            unsigned long long target = scale_exact(u, K, false);
            if (target >= K) target = K - 1;                       // u < 1; a guard, not a case
            unsigned long long cum = 0ull;
            tb = 0;
            for (int c = 0; c < a.n_chunks; ++c) {
                const int t = __ldcg(w.ctie + (long long)row * a.n_chunks + c);
                const int kt = min(t, max(0, ntie - tb));
                const unsigned long long kc = __ldcg(w.cmass + (long long)row * a.n_chunks + c) + (unsigned long long)kt * qcut;
                if (cum + kc > target) { s_chunk = c; s_before = cum; s_tb = tb; break; }
                cum += kc; tb += t;
            }
            s_target = target;
        }
        s_choice = 0x7fffffff;
    }
    __syncthreads();
    const int c = s_chunk;
    if (c >= 0) {
        // block scan of chunk c in id order: thread t owns ids base + 16 t .. + 15
        const int base = c * FCHUNK + tid * FPER;
        const bool block_eos = PROC && a.pr.eos >= 0 && step < a.pr.min_new;
        float z[FPER];
        int t = 0;
#pragma unroll
        for (int j = 0; j < FPER; ++j) {
            z[j] = base + j < a.V ? proc_one<PROC>(a, row, base + j, block_eos) : -INFINITY;
            t += z[j] > -INFINITY && fkey(z[j]) == cut && kept(z[j], weight(z[j], M, T));
        }
        int tall;
        int rank = s_tb + block_excl_scan<int>(t, s_i32, &tall);
        unsigned long long q[FPER], m = 0ull;
#pragma unroll
        for (int j = 0; j < FPER; ++j) {
            const double e = weight(z[j], M, T);
            q[j] = 0ull;
            if (kept(z[j], e)) {
                if (fkey(z[j]) != cut) q[j] = fixmass(e);
                else q[j] = (rank++ < ntie) ? fixmass(e) : 0ull;
            }
            m += q[j];
        }
        unsigned long long mall;
        unsigned long long acc = s_before + block_excl_scan<unsigned long long>(m, s_u64, &mall);
        const unsigned long long target = s_target;
        if (acc <= target && acc + m > target) {
#pragma unroll
            for (int j = 0; j < FPER; ++j) {
                acc += q[j];
                if (acc > target) { s_choice = base + j; break; }
            }
        }
    }
    __syncthreads();
    const long long choice = empty ? pad_id : (long long)s_choice;
    float lse = 0.f;
    if constexpr (LOGP) {
        if (tid < 32) {                                            // sampler.cu's combine of the two-stage chunk statistics
            const int lane = tid;
            const float2* sp = w.stats + (long long)row * a.n_chunks;
            float m = -INFINITY;
            for (int cc = lane; cc < a.n_chunks; cc += 32) m = fmaxf(m, __ldcg(&sp[cc].x));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float s = 0.f;
            for (int cc = lane; cc < a.n_chunks; cc += 32) { const float2 p = __ldcg(sp + cc); s += p.y * expf(p.x - m); }
            lse = m + logf(br::warp_sum(s));
        }
    }
    if (tid == 0) {
        const int fin = finished ? __ldcg(finished + row) : 0;
        const long long tok = fin ? pad_id : choice;
        if (tokens && step < max_steps) tokens[(long long)row * max_steps + step] = tok;
        if constexpr (LOGP) {
            if (step < max_steps) {
                const float zc = (choice >= 0 && choice < a.V) ? __ldcg(a.logits + (long long)row * a.ld + choice) : -INFINITY;
                logp[(long long)row * max_steps + step] = fin ? 0.f : zc - lse;
            }
        }
        if (next_ids) next_ids[row] = tok;
        if (finished && !fin && eos_id >= 0 && tok == eos_id) finished[row] = 1;
        if constexpr (PROC) {
            if (a.pr.presence && tok >= 0 && tok < a.V) a.pr.presence[(long long)row * ((a.V + 31) >> 5) + (tok >> 5)] |= 1u << (tok & 31);
        }
    }
}

// workspace layout (each part 16-byte aligned)
struct FullLayout {
    int64_t sel, arrive, cmax, stats, cmass, ctie, hcnt, hmass, total;
};
static int64_t al16(int64_t x) { return (x + 15) & ~(int64_t)15; }
static FullLayout full_layout(int R, int V) {
    const int64_t nc = (V + FCHUNK - 1) / FCHUNK;
    FullLayout L;
    int64_t o = 0;
    L.sel = o;    o = al16(o + (int64_t)R * sizeof(RowSel));
    L.arrive = o; o = al16(o + (int64_t)R * NARRIVE * sizeof(int));
    L.cmax = o;   o = al16(o + (int64_t)R * nc * sizeof(float));
    L.stats = o;  o = al16(o + (int64_t)R * nc * sizeof(float2));
    L.cmass = o;  o = al16(o + (int64_t)R * nc * sizeof(unsigned long long));
    L.ctie = o;   o = al16(o + (int64_t)R * nc * sizeof(int));
    L.hcnt = o;   o = al16(o + (int64_t)R * FBINS2 * sizeof(int));
    L.hmass = o;  o = al16(o + (int64_t)R * FBINS2 * sizeof(unsigned long long));
    L.total = o;
    return L;
}

template <bool LOGP, bool PROC>
static int launch_full(const FullArgs& a, const FullWs& w, int R, bool topk_on, bool topp_on, const float* uniforms, const int32_t* step,
                       int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished, int64_t* tokens, int64_t* next_ids, float* logp,
                       cudaStream_t st) {
    const dim3 grid(a.n_chunks, R), block(FTHREADS);
    BR_CHECK_CUDA(br_launch_pdl(full_stats_kernel<LOGP, PROC>, grid, block, 0, st, a, w));
    int slot = 0;
    if (topk_on)
        for (int p = 0; p < 3; ++p) BR_CHECK_CUDA(br_launch_pdl(full_select_kernel<PROC, false>, grid, block, 0, st, a, w, p, slot++));
    if (topp_on)
        for (int p = 0; p < 3; ++p) BR_CHECK_CUDA(br_launch_pdl(full_select_kernel<PROC, true>, grid, block, 0, st, a, w, p, slot++));
    BR_CHECK_CUDA(br_launch_pdl(full_draw_kernel<LOGP, PROC>, grid, block, 0, st, a, w, slot, uniforms, (const int*)step, R, max_steps,
                                (long long)eos_id, (long long)pad_id, (int*)finished, (long long*)tokens, (long long*)next_ids, logp));
    return BR_OK;
}

}  // namespace

extern "C" {

int64_t br_sample_full_workspace_bytes(int R, int V) {
    if (R <= 0 || V <= 0) return 0;
    return full_layout(R, V).total;
}

int br_sample_next_full(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, const float* uniforms,
                        const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished, int64_t* tokens,
                        int64_t* next_ids, float* logp, const br_sample_proc* proc, void* workspace, void* stream) {
    BR_CHECK_ARG(R > 0 && R <= 65535 && V > 0 && V < (1 << 23) && logits && workspace,
                 "sample_next_full: need 1 <= R <= 65535, 1 <= V < 2^23, logits and a workspace");
    BR_CHECK_ARG(temperature > 0.f && top_k >= 0 && top_p > 0.f && uniforms,
                 "sample_next_full: need T > 0, top_k >= 0, top_p > 0 and a uniforms buffer");
    Proc pr{};
    if (proc) {
        const int rc = proc_args(proc, eos_id, step, "sample_next_full", &pr);
        if (rc != BR_OK) return rc;
    }
    const FullLayout L = full_layout(R, V);
    char* b = (char*)workspace;
    const FullWs w{(RowSel*)(b + L.sel), (int*)(b + L.arrive), (float*)(b + L.cmax), (float2*)(b + L.stats),
                   (unsigned long long*)(b + L.cmass), (int*)(b + L.ctie), (int*)(b + L.hcnt), (unsigned long long*)(b + L.hmass)};
    const FullArgs a{logits, (long long)ld, V, (V + FCHUNK - 1) / FCHUNK, temperature, top_k, top_p, pr};
    const bool topk_on = top_k >= 1 && top_k < V, topp_on = top_p < 1.f;
    cudaStream_t st = (cudaStream_t)stream;
    if (logp)
        return proc ? launch_full<true, true>(a, w, R, topk_on, topp_on, uniforms, step, max_steps, eos_id, pad_id, finished, tokens, next_ids, logp, st)
                    : launch_full<true, false>(a, w, R, topk_on, topp_on, uniforms, step, max_steps, eos_id, pad_id, finished, tokens, next_ids, logp, st);
    return proc ? launch_full<false, true>(a, w, R, topk_on, topp_on, uniforms, step, max_steps, eos_id, pad_id, finished, tokens, next_ids, nullptr, st)
                : launch_full<false, false>(a, w, R, topk_on, topp_on, uniforms, step, max_steps, eos_id, pad_id, finished, tokens, next_ids, nullptr, st);
}

}  // extern "C"
