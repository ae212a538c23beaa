// Fused next-token sampler for the rollout: temperature -> top-k -> top-p -> draw, plus EOS / pad bookkeeping, one CTA
// per row, no host round trip.  Replaces the HF logits warpers + softmax + torch.multinomial / argmax and the
// unfinished_sequences bookkeeping (HF generation/utils.py:1214-1223, 2762-2797; grpo_trainer.py:384-391).
//
// top-k threshold: exact radix select over the order-preserving uint32 image of the fp32 logits (3 histogram passes
// of 11/11/10 bits, 151 936 logits stay L2-resident), ties at the threshold are all kept like HF's
// `scores < topk(scores)[..., -1]`.  top-p follows TopPLogitsWarper (ascending cumulative sum, drop while
// cum <= 1 - p, always keep the best).  The draw is inverse-CDF over the kept tokens in ascending token id with a
// caller-supplied uniform per (step, row): torch.multinomial's Philox consumption cannot be reproduced outside
// torch, so parity is defined on supplied uniforms (SURVEY.md §7 "Sampling parity").
// The *_proc entry points add HF's repetition penalty and min_new_tokens ahead of the warpers and min-p after top-p (see Proc in sampler_common.cuh).
#include "sampler_common.cuh"
#include "../../include/bioreason_b200.h"

namespace {

constexpr int MAXC = 1024;

// find bin b (descending scan) such that count(bins > b) < k <= count(bins >= b); returns b and updates k_rem
__device__ int find_bin(const int* hist, int nbins, int& k_rem, int* s_tmp) {
    // executed by warp 0; nbins multiple of 32
    const int lane = threadIdx.x & 31;
    const int per = nbins / 32;
    const int hi = nbins - 1 - lane * per;                      // lane 0 owns the top chunk
    int sum = 0;
    for (int i = 0; i < per; ++i) sum += hist[hi - i];
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    const int excl = incl - sum;
    const bool mine = (excl < k_rem) && (incl >= k_rem);
    if (mine) {
        int acc = excl, b = hi;
        for (int i = 0; i < per; ++i) {
            b = hi - i;
            if (acc + hist[b] >= k_rem) break;
            acc += hist[b];
        }
        s_tmp[0] = b; s_tmp[1] = k_rem - acc;
    }
    __syncwarp();
    int b = s_tmp[0];
    k_rem = s_tmp[1];
    return b;
}

// Fast selection of a SUPERSET of the k largest values (the common case; exactness comes from the consumer, which ranks the superset):
// one shared-memory histogram over the distance to the maximum, bin = floor((max - v) * 32) -- monotone in v, so "all elements in bins
// <= b*" (b* = the bin holding the k-th largest) contains the k largest and every tie of the k-th.  The exact 3-pass radix select over
// the raw key bits (below) puts ~all logits of a chunk into a handful of exponent bins in its first pass (serialised shared-memory
// atomics) and needs three histogram rounds; this needs one, with the counts spread over ~100 bins.  Values further than 64 below the
// maximum are not counted (they can only matter when k exceeds everything closer, which falls back to the radix select).
constexpr int FBINS = 2048;
constexpr float FBIN_SCALE = 32.f;
__device__ __forceinline__ int fast_bin(float mx, float v) {
    const float d = (mx - v) * FBIN_SCALE;                       // NaN (mx = v = -inf) -> 0, +inf -> saturates
    return d >= (float)(FBINS - 1) ? FBINS - 1 : __float2int_rd(d);
}
// warp 0: smallest bin b with count(bins <= b) >= k -> out[0] = b (or -1), out[1] = count(bins <= b)
__device__ void find_bin_asc(const int* hist, int k, int* out) {
    const int lane = threadIdx.x & 31;
    int acc = 0, found = -1, cnt = 0;
    for (int base = 0; base < FBINS - 32; base += 32) {          // the last bin (saturated values) is never counted
        const int c = hist[base + lane];
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (acc + total >= k) {
            const unsigned m = __ballot_sync(0xffffffffu, acc + incl >= k);
            const int l = __ffs(m) - 1;
            found = base + l; cnt = acc + __shfl_sync(0xffffffffu, incl, l);
            break;
        }
        acc += total;
    }
    if (lane == 0) { out[0] = found; out[1] = cnt; }
}

// Behaviour log-prob (the *_logp entry points): logp[r, step] = z[y] - logsumexp(z) over the raw fp32 logits of the row (T = 1, the
// full vocabulary) -- the quantity br_lmhead_logprob_fwd gives the scoring passes.  Two-stage path: stage 1 writes each chunk's
// (max m_c, sum exp(z - m_c)), stage 2 combines the pairs in chunk order; single stage: a block-wide LSE over the row.

// Stage 1 (many CTAs): each CTA owns a 4096-logit chunk of one row, keeps it in registers, finds the chunk's exact
// top_k-th value by radix select on shared-memory histograms and emits every element >= that value (value, token id) --
// a superset of the row's global top-k.  Stage 2 (sampler_kernel, one CTA per row) then works on <= chunks*CAND_CAP
// candidates instead of 151 936 logits: the sampler drops from ~200 us to ~20 us per decode step.
// A chunk holding more than CAND_CAP finite values >= its k-th (only ties of the k-th can do that) emits the lowest-id CAND_CAP
// and sets its overflow flag; stage 2 then selects on the logits row itself, so no tie HF keeps is lost.
constexpr int CHUNK = 4096, CAND_CAP = 64;

// Processed path (the *_proc entry points, PROC = true): Proc and proc_logit in sampler_common.cuh.

template <bool LOGP, bool PROC>
__global__ void __launch_bounds__(256, 1) sampler_partial_kernel(const float* __restrict__ logits, long long ld, int V, int top_k,
                                                              float* __restrict__ cand_val, int* __restrict__ cand_idx, int n_chunks,
                                                              int* __restrict__ overflow, float2* __restrict__ chunk_stats, Proc pr) {
    __shared__ int hist[2048];
    __shared__ int s_tmp[4];
    __shared__ int s_count, s_ties;
    const int chunk = blockIdx.x, row = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    br::launch_dependents();
    br::grid_dep_wait();
    const float* x = logits + (long long)row * ld;
    const int base = chunk * CHUNK;
    float v[16]; uint32_t key[16];
    int n_valid = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int idx = base + i * 256 + tid;
        const bool ok = idx < V;
        v[i] = ok ? __ldcg(x + idx) : -INFINITY;          // L2 loads throughout: PDL-chained kernels keep no coherent L1
        key[i] = ok ? fkey(v[i]) : 0u;
        n_valid += ok;
    }
    if constexpr (PROC) {
        if constexpr (LOGP) {
            // the chunk statistics of the log-prob come from the raw values
            __shared__ float s_red_raw[32];
            float mr = -INFINITY;
#pragma unroll
            for (int i = 0; i < 16; ++i) mr = fmaxf(mr, v[i]);
            mr = block_max(mr, s_red_raw);
            float s = 0.f;
            if (mr > -INFINITY) {
#pragma unroll
                for (int i = 0; i < 16; ++i) s += expf(v[i] - mr);
            }
            s = block_sum(s, s_red_raw);
            if (tid == 0) chunk_stats[(long long)row * n_chunks + chunk] = make_float2(mr, s);
        }
        // a warp's 32 consecutive ids share one bitmap word: one broadcast load per i
        const int step = pr.step ? __ldcg(pr.step) : 0;
        const bool block_eos = pr.eos >= 0 && step < pr.min_new;
        const uint32_t* pres = pr.presence ? pr.presence + (long long)row * ((V + 31) >> 5) : nullptr;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int idx = base + i * 256 + tid;
            if (idx < V) {
                v[i] = proc_logit(v[i], proc_in_set(pres, idx), block_eos && idx == pr.eos, pr.theta);
                key[i] = fkey(v[i]);
            }
        }
    }
    const int n_here = min(CHUNK, V - base);
    const int k = min(top_k, n_here);
    float* cv = cand_val + ((long long)row * n_chunks + chunk) * CAND_CAP;
    int* ci = cand_idx + ((long long)row * n_chunks + chunk) * CAND_CAP;
    // ---- fast path: one histogram over the distance to the chunk maximum (see fast_bin)
    {
        __shared__ float s_red[32];
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < 16; ++i) mx = fmaxf(mx, v[i]);
        mx = block_max(mx, s_red);
        if constexpr (LOGP && !PROC) {
            // (m_c, s_c) before the fast / exact split (the fast path returns early); entries past V hold -inf and add 0, and an
            // all -inf chunk gives (-inf, 0)
            float s = 0.f;
            if (mx > -INFINITY) {
#pragma unroll
                for (int i = 0; i < 16; ++i) s += expf(v[i] - mx);
            }
            s = block_sum(s, s_red);
            if (tid == 0) chunk_stats[(long long)row * n_chunks + chunk] = make_float2(mx, s);
        }
        for (int i = tid; i < FBINS; i += 256) hist[i] = 0;
        if (tid == 0) s_count = 0;
        __syncthreads();
        int bin[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            bin[i] = (base + i * 256 + tid < V) ? fast_bin(mx, v[i]) : FBINS - 1;
            if (bin[i] < FBINS - 1) atomicAdd(&hist[bin[i]], 1);
        }
        __syncthreads();
        if (warp == 0) find_bin_asc(hist, k, s_tmp);
        __syncthreads();
        const int bstar = s_tmp[0], cnt = s_tmp[1];
        if (mx > -INFINITY && bstar >= 0 && cnt <= CAND_CAP) {                  // uniform across the CTA
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (bin[i] <= bstar) {
                    const int s = atomicAdd(&s_count, 1);
                    cv[s] = v[i]; ci[s] = base + i * 256 + tid;
                }
            }
            for (int s = cnt + tid; s < CAND_CAP; s += 256) { cv[s] = -INFINITY; ci[s] = 0x7fffffff; }
            if (tid == 0) overflow[(long long)row * n_chunks + chunk] = 0;
            return;
        }
        __syncthreads();
    }
    // ---- exact path (degenerate chunks: > CAND_CAP values within 1/32 of the k-th, or nothing finite)
    uint32_t prefix = 0; int k_rem = k;
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
        const int nb = pass == 2 ? 1024 : 2048;
        for (int i = tid; i < 2048; i += 256) hist[i] = 0;
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int idx = base + i * 256 + tid;
            if (idx < V) {
                bool in;
                if (pass == 0) in = true; else if (pass == 1) in = (key[i] >> 21) == prefix; else in = (key[i] >> 10) == prefix;
                if (in) atomicAdd(&hist[(key[i] >> shift) & (nb - 1)], 1);
            }
        }
        __syncthreads();
        if (warp == 0) {
            int kr = k_rem;
            int b = find_bin(hist, nb, kr, s_tmp);
            if (lane == 0) { s_tmp[2] = b; s_tmp[3] = kr; }
        }
        __syncthreads();
        const int b = s_tmp[2];
        k_rem = s_tmp[3];
        prefix = pass == 0 ? (uint32_t)b : (pass == 1 ? ((prefix << 11) | (uint32_t)b) : ((prefix << 10) | (uint32_t)b));
        __syncthreads();
    }
    // values strictly above the k-th (fewer than k) always fit; ties OF the k-th fill the remaining slots in token-id order, so the
    // emitted set does not depend on the order in which threads reach an atomic
    if (tid == 0) { s_count = 0; s_ties = 0; }
    __syncthreads();
    int my_ties = 0;                                                   // finite ties only: -inf is never kept
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int idx = base + i * 256 + tid;
        if (idx < V && key[i] > prefix) {
            const int s = atomicAdd(&s_count, 1);
            if (s < CAND_CAP) { cv[s] = v[i]; ci[s] = idx; }
        }
        my_ties += idx < V && key[i] == prefix && v[i] > -INFINITY;
    }
    if (my_ties) atomicAdd(&s_ties, my_ties);
    __syncthreads();
    if (tid == 0) overflow[(long long)row * n_chunks + chunk] = s_count + s_ties > CAND_CAP;
    int filled = min(s_count, CAND_CAP);
    __shared__ int s_w[8];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        if (filled >= CAND_CAP) break;                                 // uniform across the CTA
        const int idx = base + i * 256 + tid;
        const bool tie = idx < V && key[i] == prefix;
        const unsigned m = __ballot_sync(0xffffffffu, tie);
        if (lane == 0) s_w[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { const int c = s_w[w]; total += c; if (w < warp) before += c; }
        const int slot = filled + before + __popc(m & ((1u << lane) - 1u));
        if (tie && slot < CAND_CAP) { cv[slot] = v[i]; ci[slot] = idx; }
        filled = min(CAND_CAP, filled + total);
        __syncthreads();
    }
    for (int s = filled + tid; s < CAND_CAP; s += 256) { cv[s] = -INFINITY; ci[s] = 0x7fffffff; }
}

// Stage 2 / single-stage sampler.  cand_idx == nullptr: x is the full logits row (index = position).
// Stage 2 also gets the logits rows themselves (row_logits, row_ld, row_V) and stage 1's per-chunk overflow flags: when a chunk
// dropped ties, or the candidates' ties of the k-th do not fit in MAXC, it selects on the row like the single-stage sampler.
// Kept set: every value above the k-th plus its ties; past MAXC values in all, the ties with the lowest token ids.
// LOGP: also writes logp[row, step]; chunk_stats = stage 1's n_chunks (m_c, s_c) pairs per row, or nullptr (single stage: x is the row).
template <bool LOGP, bool PROC>
__global__ void __launch_bounds__(1024, 1) sampler_kernel(const float* __restrict__ logits, long long ld, int V, const int* __restrict__ cand_idx_all,
                                                       const float* __restrict__ row_logits, long long row_ld, int row_V,
                                                       const int* __restrict__ overflow, float temperature, int top_k,
                                                       float top_p, int do_sample, const float* __restrict__ uniforms,
                                                       const int* __restrict__ step_ptr, int R, int max_steps, long long eos_id,
                                                       long long pad_id, int* __restrict__ finished, long long* __restrict__ tokens,
                                                       long long* __restrict__ next_ids, const float2* __restrict__ chunk_stats, int n_chunks,
                                                       float* __restrict__ logp, Proc pr) {
    __shared__ int hist[2048];
    __shared__ int s_tmp[4];
    __shared__ float c_val[MAXC];
    __shared__ int c_idx[MAXC];
    __shared__ float o_val[MAXC];
    __shared__ int o_idx[MAXC];
    __shared__ int s_count, s_ties;
    __shared__ float r_val[32];
    __shared__ int r_idx[32];
    __shared__ float s_chosen_z;                                       // LOGP: the chosen token's raw logit

    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    br::launch_dependents();
    br::grid_dep_wait();
    const float* x = logits + (long long)row * ld;
    const int* xi = cand_idx_all ? cand_idx_all + (long long)row * ld : nullptr;
    auto IDX = [&](int i) { return xi ? __ldcg(xi + i) : i; };
    const int step = step_ptr ? __ldcg(step_ptr) : 0;
    long long choice;
    // PROC: the row itself (single stage, or stage 2's fallback) is read through proc_logit; the candidates already carry processed values
    const int rowV = xi ? row_V : V;
    const uint32_t* pres = nullptr;
    bool block_eos = false;
    if constexpr (PROC) {
        pres = pr.presence ? pr.presence + (long long)row * ((rowV + 31) >> 5) : nullptr;
        block_eos = pr.eos >= 0 && step < pr.min_new;
    }
    auto PZ = [&](float z, int id) { return proc_logit(z, proc_in_set(pres, id), block_eos && id == pr.eos, pr.theta); };

    if (!do_sample) {
        float bv = -INFINITY; int bi = 0x7fffffff;
        for (int i = tid; i < V; i += blockDim.x) {
            float v = __ldcg(x + i); const int id = IDX(i);
            if constexpr (PROC) { if (!xi) v = PZ(v, i); }
            if (v > bv || (v == bv && id < bi)) { bv = v; bi = id; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ov = __shfl_xor_sync(0xffffffffu, bv, o); int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { r_val[warp] = bv; r_idx[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            bv = lane < (blockDim.x >> 5) ? r_val[lane] : -INFINITY; bi = lane < (blockDim.x >> 5) ? r_idx[lane] : 0x7fffffff;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                float ov = __shfl_xor_sync(0xffffffffu, bv, o); int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) s_tmp[2] = bi;
            if constexpr (LOGP) { if (lane == 0) s_chosen_z = bv; }
        }
        __syncthreads();
        choice = s_tmp[2];
    } else {
      bool fast_done = false;
      int ovf = 0;                                                     // some stage-1 chunk of this row dropped ties (uniform)
      if (xi != nullptr && V <= 4 * (int)blockDim.x) {
        // ---- fast path over the stage-1 candidates (<= 4 per thread): superset by distance-to-maximum bins, exact ranking below
        float v[4]; int id[4]; int bin[4];
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * blockDim.x;
            const bool ok = idx < V;
            v[i] = ok ? __ldcg(x + idx) : -INFINITY; id[i] = ok ? __ldcg(xi + idx) : 0x7fffffff;
            mx = fmaxf(mx, v[i]);
        }
        int f = 0;
        for (int c = tid; c < n_chunks; c += blockDim.x) f |= __ldcg(overflow + (long long)row * n_chunks + c);
        mx = block_max(mx, r_val);
        for (int i = tid; i < FBINS; i += blockDim.x) hist[i] = 0;
        if (tid == 0) s_count = 0;
        ovf = __syncthreads_or(f);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            bin[i] = v[i] > -INFINITY ? fast_bin(mx, v[i]) : FBINS - 1;
            if (bin[i] < FBINS - 1) atomicAdd(&hist[bin[i]], 1);
        }
        __syncthreads();
        if (warp == 0) find_bin_asc(hist, top_k, s_tmp);
        __syncthreads();
        const int bstar = s_tmp[0], cnt = s_tmp[1];
        __syncthreads();
        if (!ovf && mx > -INFINITY && bstar >= 0 && cnt <= MAXC) {              // uniform across the CTA
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (bin[i] <= bstar) { const int s = atomicAdd(&s_count, 1); c_val[s] = v[i]; c_idx[s] = id[i]; }
            }
            fast_done = true;
        }
        __syncthreads();
      } else if (xi != nullptr) {
        int f = 0;
        for (int c = tid; c < n_chunks; c += blockDim.x) f |= __ldcg(overflow + (long long)row * n_chunks + c);
        ovf = __syncthreads_or(f);
      }
      if (!fast_done) {
        // candidates, or the logits row itself when the candidates may lack ties of the k-th
        const float* src = x; const int* src_i = xi; int n = V;
        if (ovf) { src = row_logits + (long long)row * row_ld; src_i = nullptr; n = row_V; }
        for (;;) {                                                     // at most twice: candidates, then the row
            const int k = min(top_k, n);                               // HF clamps top_k to the vocabulary
            // ---- exact k-th largest key by 3-pass radix select
            uint32_t prefix = 0; int k_rem = k;
            for (int pass = 0; pass < 3; ++pass) {
                const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
                const int nb = pass == 2 ? 1024 : 2048;
                for (int i = tid; i < 2048; i += blockDim.x) hist[i] = 0;
                __syncthreads();
                for (int i = tid; i < n; i += blockDim.x) {
                    float zv = __ldcg(src + i);
                    if constexpr (PROC) { if (!src_i) zv = PZ(zv, i); }
                    const uint32_t key = fkey(zv);
                    bool in;
                    if (pass == 0) in = true; else if (pass == 1) in = (key >> 21) == prefix; else in = (key >> 10) == prefix;
                    if (in) atomicAdd(&hist[(key >> shift) & (nb - 1)], 1);
                }
                __syncthreads();
                if (warp == 0) {
                    int kr = k_rem;
                    int b = find_bin(hist, nb, kr, s_tmp);
                    if (lane == 0) { s_tmp[2] = b; s_tmp[3] = kr; }
                }
                __syncthreads();
                const int b = s_tmp[2];
                k_rem = s_tmp[3];
                prefix = pass == 0 ? (uint32_t)b : (pass == 1 ? ((prefix << 11) | (uint32_t)b) : ((prefix << 10) | (uint32_t)b));
                __syncthreads();
            }
            const uint32_t thr = prefix;
            // values above the k-th (fewer than k) go to the front; its ties to the back while they fit beside them
            const int tie_room = MAXC - k;
            if (tid == 0) { s_count = 0; s_ties = 0; }
            __syncthreads();
            for (int i = tid; i < n; i += blockDim.x) {
                float v = __ldcg(src + i);
                if constexpr (PROC) { if (!src_i) v = PZ(v, i); }
                if (!(v > -INFINITY)) continue;
                const uint32_t key = fkey(v);
                if (key > thr) {
                    const int s = atomicAdd(&s_count, 1);
                    c_val[s] = v; c_idx[s] = src_i ? __ldcg(src_i + i) : i;
                } else if (key == thr) {
                    const int t = atomicAdd(&s_ties, 1);
                    if (t < tie_room) { c_val[MAXC - 1 - t] = v; c_idx[MAXC - 1 - t] = src_i ? __ldcg(src_i + i) : i; }
                }
            }
            __syncthreads();
            const int n_above = s_count, n_tie = s_ties;
            if (n_tie <= tie_room) {                                   // every tie collected: move them next to the values above
                const bool mv = tid < n_tie;
                float tv = 0.f; int ti = 0;
                if (mv) { tv = c_val[MAXC - 1 - tid]; ti = c_idx[MAXC - 1 - tid]; }
                __syncthreads();
                if (mv) { c_val[n_above + tid] = tv; c_idx[n_above + tid] = ti; }
                if (tid == 0) s_count = n_above + n_tie;
                __syncthreads();
                break;
            }
            if (src_i == nullptr) {
                // more ties than room (the row itself: index = token id): fill with the lowest-id ties, so the kept set does not
                // depend on the order in which threads reach an atomic
                __shared__ int s_w[32];
                const int nw = blockDim.x >> 5;
                int filled = n_above;
                for (int base = 0; base < n && filled < MAXC; base += blockDim.x) {       // uniform across the CTA
                    const int i = base + tid;
                    float v = i < n ? __ldcg(src + i) : -INFINITY;
                    if constexpr (PROC) { if (i < n) v = PZ(v, i); }
                    const bool tie = v > -INFINITY && fkey(v) == thr;
                    const unsigned m = __ballot_sync(0xffffffffu, tie);
                    if (lane == 0) s_w[warp] = __popc(m);
                    __syncthreads();
                    int before = 0, total = 0;
                    for (int w = 0; w < nw; ++w) { const int c = s_w[w]; total += c; if (w < warp) before += c; }
                    const int slot = filled + before + __popc(m & ((1u << lane) - 1u));
                    if (tie && slot < MAXC) { c_val[slot] = v; c_idx[slot] = i; }
                    filled = min(MAXC, filled + total);
                    __syncthreads();
                }
                if (tid == 0) s_count = filled;
                __syncthreads();
                break;
            }
            src = row_logits + (long long)row * row_ld; src_i = nullptr; n = row_V;   // candidate ties do not fit: select on the row
        }
      }
        const int c_all = min(s_count, MAXC);
        // ---- rank sort: descending value, ties by ascending index
        if (tid < c_all) {
            const float v = c_val[tid]; const int id = c_idx[tid];
            int rank = 0;
            for (int j = 0; j < c_all; ++j) rank += (c_val[j] > v) || (c_val[j] == v && c_idx[j] < id);
            o_val[rank] = v; o_idx[rank] = id;
        }
        __syncthreads();
        if (tid == 0) {
            // top-k with HF's tie rule (`scores < topk(scores)[..., -1]` are dropped: every value equal to the k-th stays); the
            // collected set may be a superset (fast path) or exactly that set (radix path)
            int c = min(top_k, c_all);
            if (c > 0) { const float kth = o_val[c - 1]; while (c < c_all && o_val[c] == kth) ++c; }
            // softmax over the kept-by-top-k set at temperature T (fp32), descending order
            const float inv_t = 1.f / temperature;
            const float mx = o_val[0] * inv_t;
            float tot = 0.f;
            for (int j = 0; j < c; ++j) { c_val[j] = __expf(o_val[j] * inv_t - mx); tot += c_val[j]; }
            // top-p: ascending cumulative sum; drop while cum <= 1 - p; the best token always stays
            int keep = c;
            if (top_p < 1.f) {
                float cum = 0.f;
                const float lim = 1.f - top_p;
                for (int j = c - 1; j >= 1; --j) {
                    cum += c_val[j] / tot;
                    if (cum <= lim) keep = j; else break;
                }
            }
            if constexpr (PROC) {
                // min-p (HF MinPLogitsWarper, after top-p): drop p_j < min_p p_max, i.e. e_j = exp((z_j - z_max) / T) < min_p; the
                // maximum always stays
                if (pr.min_p > 0.f) {
                    for (int j = 1; j < keep; ++j) if (c_val[j] < pr.min_p) { keep = j; break; }
                }
            }
            float ktot = 0.f;
            for (int j = 0; j < keep; ++j) ktot += c_val[j];
            // inverse CDF in ascending token id
            const float u = uniforms[(long long)step * R + row];
            const float target = u * ktot;
            // selection by repeatedly taking the smallest remaining id (keep is ~20)
            float acc = 0.f; int chosen = o_idx[0]; int last_id = -1;
            float chosen_z = o_val[0];
            for (int n = 0; n < keep; ++n) {
                int best = -1;
                for (int j = 0; j < keep; ++j) if (o_idx[j] > last_id && (best < 0 || o_idx[j] < o_idx[best])) best = j;
                acc += c_val[best]; last_id = o_idx[best]; chosen = o_idx[best];
                if constexpr (LOGP) chosen_z = o_val[best];
                if (acc > target) break;
            }
            s_tmp[2] = chosen;
            if constexpr (LOGP) s_chosen_z = chosen_z;
        }
        __syncthreads();
        choice = s_tmp[2];
    }
    float lse = 0.f;                                                   // valid in thread 0
    if constexpr (LOGP) {
        if (chunk_stats) {
            if (warp == 0) {
                const float2* st = chunk_stats + (long long)row * n_chunks;
                float m = -INFINITY;
                for (int c = lane; c < n_chunks; c += 32) m = fmaxf(m, __ldcg(&st[c].x));
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                float s = 0.f;
                for (int c = lane; c < n_chunks; c += 32) { const float2 p = __ldcg(st + c); s += p.y * expf(p.x - m); }
                lse = m + logf(br::warp_sum(s));
            }
        } else {
            float m = -INFINITY;
            for (int i = tid; i < V; i += blockDim.x) m = fmaxf(m, __ldcg(x + i));
            m = block_max(m, r_val);
            float s = 0.f;
            if (m > -INFINITY) for (int i = tid; i < V; i += blockDim.x) s += expf(__ldcg(x + i) - m);
            lse = m + logf(block_sum(s, r_val));
        }
    }
    if constexpr (LOGP && PROC) {
        if (tid == 0) {                                                // the log-prob reads the raw logit of the chosen token
            const float* zr = xi ? row_logits + (long long)row * row_ld : x;
            s_chosen_z = (choice >= 0 && choice < rowV) ? __ldcg(zr + choice) : -INFINITY;
        }
    }
    if (tid == 0) {
        const int fin = finished ? __ldcg(finished + row) : 0;
        long long tok = fin ? pad_id : choice;                         // finished rows emit pad (HF :2796-2797)
        if (tokens && step < max_steps) tokens[(long long)row * max_steps + step] = tok;
        if constexpr (LOGP) { if (step < max_steps) logp[(long long)row * max_steps + step] = fin ? 0.f : s_chosen_z - lse; }
        if (next_ids) next_ids[row] = tok;
        if (finished && !fin && eos_id >= 0 && tok == eos_id) finished[row] = 1;
        if constexpr (PROC) {
            if (pr.presence && tok >= 0 && tok < rowV) pr.presence[(long long)row * ((rowV + 31) >> 5) + (tok >> 5)] |= 1u << (tok & 31);
        }
    }
}

__global__ void advance_kernel(int* step, int* cur_len, int R) {
    const int i = threadIdx.x;
    // NO early launch_dependents() here: this kernel is the token-step boundary.  Later kernels of the chain (the fused decode
    // attention) read cur_len BEFORE their own dependency wait; keeping the implicit trigger at completion guarantees that nothing
    // of step N+1 starts before cur_len of step N is final (and, transitively, before every kernel of step N has completed).
    br::grid_dep_wait();
    if (i < R) atomicAdd(cur_len + i, 1);
    if (i == 0 && step) atomicAdd(step, 1);
}

}  // namespace

extern "C" {

int br_sample_next(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                   const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                   int64_t* tokens, int64_t* next_ids, void* stream) {
    BR_CHECK_ARG(R > 0 && V > 0, "sample_next: empty");
    if (do_sample) {
        BR_CHECK_ARG(temperature > 0.f && top_k >= 1 && top_k <= MAXC && top_p > 0.f && uniforms, "sample_next: need T > 0, 1 <= top_k <= %d, top_p > 0 and a uniforms buffer", MAXC);
    }
    sampler_kernel<false, false><<<R, 1024, 0, (cudaStream_t)stream>>>(logits, ld, V, nullptr, nullptr, 0, 0, nullptr, temperature, top_k, top_p, do_sample, uniforms, step, R, max_steps,
                                                                      (long long)eos_id, (long long)pad_id, finished, (long long*)tokens, (long long*)next_ids,
                                                                      nullptr, 0, nullptr, Proc{});
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_sample_next_logp(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                        const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                        int64_t* tokens, int64_t* next_ids, float* logp, void* stream) {
    BR_CHECK_ARG(R > 0 && V > 0 && logp, "sample_next_logp: empty / no logp buffer");
    if (do_sample) {
        BR_CHECK_ARG(temperature > 0.f && top_k >= 1 && top_k <= MAXC && top_p > 0.f && uniforms, "sample_next_logp: need T > 0, 1 <= top_k <= %d, top_p > 0 and a uniforms buffer", MAXC);
    }
    sampler_kernel<true, false><<<R, 1024, 0, (cudaStream_t)stream>>>(logits, ld, V, nullptr, nullptr, 0, 0, nullptr, temperature, top_k, top_p, do_sample, uniforms, step, R, max_steps,
                                                                     (long long)eos_id, (long long)pad_id, finished, (long long*)tokens, (long long*)next_ids,
                                                                     nullptr, 0, logp, Proc{});
    BR_CHECK_LAUNCH();
    return BR_OK;
}

// workspace: candidate values and ids [R, n_chunks, CAND_CAP], then the chunks' overflow flags [R, n_chunks] (int, padded to 8 bytes)
static int64_t flag_ints(int R, int n_chunks) { return ((int64_t)R * n_chunks + 1) & ~(int64_t)1; }

int64_t br_sample_workspace_bytes(int R, int V) {
    const int n_chunks = (V + CHUNK - 1) / CHUNK;
    return (int64_t)R * n_chunks * CAND_CAP * (sizeof(float) + sizeof(int)) + flag_ints(R, n_chunks) * sizeof(int);
}

int64_t br_sample_logp_workspace_bytes(int R, int V) {
    const int n_chunks = (V + CHUNK - 1) / CHUNK;
    return br_sample_workspace_bytes(R, V) + (int64_t)R * n_chunks * sizeof(float2);
}

}  // extern "C"

template <bool PROC>
static int sample_2stage(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                         const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                         int64_t* tokens, int64_t* next_ids, float* logp, void* workspace, void* stream, Proc pr = Proc{}) {
    BR_CHECK_ARG(R > 0 && V > 0 && workspace, "sample_next_2stage: empty / no workspace");
    const int k = do_sample ? top_k : 1;
    BR_CHECK_ARG(k >= 1 && k <= CAND_CAP / 2, "sample_next_2stage: top_k must be in [1, %d]", CAND_CAP / 2);
    if (do_sample) BR_CHECK_ARG(temperature > 0.f && top_p > 0.f && uniforms, "sample_next_2stage: need T > 0, top_p > 0 and a uniforms buffer");
    const int n_chunks = (V + CHUNK - 1) / CHUNK;
    float* cv = (float*)workspace;
    int* ci = (int*)(cv + (int64_t)R * n_chunks * CAND_CAP);
    cudaStream_t st = (cudaStream_t)stream;
    int* flags = ci + (int64_t)R * n_chunks * CAND_CAP;
    const int n_cand = n_chunks * CAND_CAP;
    if (!logp) {
        BR_CHECK_CUDA(br_launch_pdl(sampler_partial_kernel<false, PROC>, dim3(n_chunks, R), dim3(256), 0, st, logits, (long long)ld, V, k, cv, ci, n_chunks,
                                    flags, (float2*)nullptr, pr));
        BR_CHECK_CUDA(br_launch_pdl(sampler_kernel<false, PROC>, dim3(R), dim3(1024), 0, st, (const float*)cv, (long long)n_cand, n_cand, (const int*)ci,
                                    logits, (long long)ld, V, (const int*)flags,
                                    temperature, top_k, top_p, do_sample, uniforms, step, R, max_steps, (long long)eos_id, (long long)pad_id,
                                    finished, (long long*)tokens, (long long*)next_ids, (const float2*)nullptr, n_chunks, (float*)nullptr, pr));
        return BR_OK;
    }
    float2* stats = (float2*)(flags + flag_ints(R, n_chunks));             // the tail of br_sample_logp_workspace_bytes
    BR_CHECK_CUDA(br_launch_pdl(sampler_partial_kernel<true, PROC>, dim3(n_chunks, R), dim3(256), 0, st, logits, (long long)ld, V, k, cv, ci, n_chunks,
                                flags, stats, pr));
    BR_CHECK_CUDA(br_launch_pdl(sampler_kernel<true, PROC>, dim3(R), dim3(1024), 0, st, (const float*)cv, (long long)n_cand, n_cand, (const int*)ci,
                                logits, (long long)ld, V, (const int*)flags,
                                temperature, top_k, top_p, do_sample, uniforms, step, R, max_steps, (long long)eos_id, (long long)pad_id,
                                finished, (long long*)tokens, (long long*)next_ids, (const float2*)stats, n_chunks, logp, pr));
    return BR_OK;
}

extern "C" {

/* two-stage variant for large vocabularies (same semantics as br_sample_next) */
int br_sample_next_2stage(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                          const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                          int64_t* tokens, int64_t* next_ids, void* workspace, void* stream) {
    return sample_2stage<false>(logits, ld, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                                next_ids, nullptr, workspace, stream);
}

int br_sample_next_2stage_logp(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                               const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                               int64_t* tokens, int64_t* next_ids, float* logp, void* workspace, void* stream) {
    BR_CHECK_ARG(logp, "sample_next_2stage_logp: no logp buffer");
    return sample_2stage<false>(logits, ld, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                                next_ids, logp, workspace, stream);
}

int br_sample_next_proc(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                        const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                        int64_t* tokens, int64_t* next_ids, float* logp, const br_sample_proc* proc, void* stream) {
    BR_CHECK_ARG(R > 0 && V > 0, "sample_next_proc: empty");
    if (do_sample) {
        BR_CHECK_ARG(temperature > 0.f && top_k >= 1 && top_k <= MAXC && top_p > 0.f && uniforms, "sample_next_proc: need T > 0, 1 <= top_k <= %d, top_p > 0 and a uniforms buffer", MAXC);
    }
    Proc pr;
    const int rc = proc_args(proc, eos_id, step, "sample_next_proc", &pr);
    if (rc != BR_OK) return rc;
    if (logp) {
        sampler_kernel<true, true><<<R, 1024, 0, (cudaStream_t)stream>>>(logits, ld, V, nullptr, nullptr, 0, 0, nullptr, temperature, top_k, top_p, do_sample, uniforms, step, R,
                                                                        max_steps, (long long)eos_id, (long long)pad_id, finished, (long long*)tokens,
                                                                        (long long*)next_ids, nullptr, 0, logp, pr);
    } else {
        sampler_kernel<false, true><<<R, 1024, 0, (cudaStream_t)stream>>>(logits, ld, V, nullptr, nullptr, 0, 0, nullptr, temperature, top_k, top_p, do_sample, uniforms, step, R,
                                                                         max_steps, (long long)eos_id, (long long)pad_id, finished, (long long*)tokens,
                                                                         (long long*)next_ids, nullptr, 0, nullptr, pr);
    }
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_sample_next_2stage_proc(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                               const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                               int64_t* tokens, int64_t* next_ids, float* logp, const br_sample_proc* proc, void* workspace, void* stream) {
    Proc pr;
    const int rc = proc_args(proc, eos_id, step, "sample_next_2stage_proc", &pr);
    if (rc != BR_OK) return rc;
    return sample_2stage<true>(logits, ld, R, V, temperature, top_k, top_p, do_sample, uniforms, step, max_steps, eos_id, pad_id, finished, tokens,
                               next_ids, logp, workspace, stream, pr);
}

int br_decode_advance(int32_t* step, int32_t* cur_len, int R, void* stream) {
    BR_CHECK_ARG(R > 0 && R <= 1024, "decode_advance: R in [1, 1024]");
    BR_CHECK_CUDA(br_launch_pdl(advance_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, step, cur_len, R));
    return BR_OK;
}

}  // extern "C"
