// Entropy threshold of the GRPO token selection ("Beyond the 80/20 Rule", TRL's top_entropy_quantile):
//   tau = torch.quantile(x[mask != 0], q)   (linear interpolation), bit for bit, without a host sync.
// torch sorts the n valid values, takes r = q * (n - 1) in fp32, the order statistics at floor(r) and ceil(r), and interpolates them
// with its lerp rule (weight w = r - floor(r); a + w (b - a) for w < 0.5, b - (b - a)(1 - w) otherwise, each one fused multiply-add).
// Here the two order statistics come from an exact radix select over the order-preserving uint32 image of the fp32 values: four
// 8-bit histogram passes find the floor(r)-th key; the ceil(r)-th is the same key while ties of it remain, else the least larger key
// (one more pass).  One CTA: n is at most world x rows x completion length, a few million at most, read five times.
// Masked entries are never read as values, so whatever they hold (NaN included) does not matter.  No valid entry: tau = +inf (every
// token is dropped, like TRL's all-false mask).  A NaN among the valid values makes tau NaN, as in torch.  -0 is read as +0.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

namespace {

constexpr int NT = 1024;

__device__ __forceinline__ uint32_t order_key(float x) {
    if (x == 0.f) x = 0.f;                                              // -0 -> +0
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_value(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// warp-aggregated shared-memory histogram add: lanes with the same bin add once
__device__ __forceinline__ void hist_add(unsigned int* hist, uint32_t bin, bool active) {
    const unsigned int act = __ballot_sync(0xffffffffu, active);
    if (!active) return;
    const unsigned int peers = __match_any_sync(act, bin);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[bin], (unsigned int)__popc(peers));
}

__global__ void __launch_bounds__(NT, 1) entropy_threshold_kernel(const float* __restrict__ x, const int* __restrict__ mask, long long n,
                                                                  float q, float* __restrict__ tau) {
    __shared__ unsigned int hist[256];
    __shared__ unsigned int s_prefix, s_nvalid, s_rank, s_eq, s_min_above, s_nan;
    if (threadIdx.x == 0) s_nan = 0u;
    uint32_t prefix = 0;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        for (int i = threadIdx.x; i < 256; i += NT) hist[i] = 0;
        __syncthreads();
        // every thread of a warp walks the loop the same number of times, so the warp-wide ballot in hist_add is uniform
        const long long n_round = (n + 31) & ~31ll;
        for (long long i = threadIdx.x; i < n_round; i += NT) {
            bool ok = i < n && mask[i] != 0;
            uint32_t k = ok ? order_key(x[i]) : 0u;
            if (pass > 0) ok = ok && (k >> (shift + 8)) == prefix;
            hist_add(hist, (k >> shift) & 255u, ok);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (pass == 0) {
                unsigned int nv = 0;
                for (int b = 0; b < 256; ++b) nv += hist[b];
                s_nvalid = nv;
                if (nv > 0) s_rank = (unsigned int)(q * (float)(nv - 1));     // floor(r), r = q (fp32) * last_index as torch forms it
            }
            if (s_nvalid > 0) {
                unsigned int k = s_rank, b = 0;
                while (k >= hist[b]) { k -= hist[b]; ++b; }
                s_rank = k;                                              // rank within the keys that share the prefix so far
                s_eq = hist[b];
                s_prefix = (prefix << 8) | b;
            }
        }
        __syncthreads();
        if (s_nvalid == 0) {
            if (threadIdx.x == 0) tau[0] = INFINITY;
            return;
        }
        prefix = s_prefix;
    }
    // prefix = key of the floor(r)-th value; s_eq valid values share it, s_rank of them come before it in sorted order.
    // The ceil(r)-th value is the same key while a tie of it follows, else the least larger key (NaN keys lie above +inf).
    if (threadIdx.x == 0) s_min_above = 0xffffffffu;
    __syncthreads();
    unsigned int m = 0xffffffffu;
    bool has_nan = false;
    for (long long i = threadIdx.x; i < n; i += NT) {
        if (mask[i] == 0) continue;
        const float v = x[i];
        const uint32_t k = order_key(v);
        has_nan |= v != v;
        if (k > prefix && k < m) m = k;
    }
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    has_nan = __any_sync(0xffffffffu, has_nan);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&s_min_above, m);
        if (has_nan) s_nan = 1u;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float lo = key_value(prefix);
        const float r = q * (float)(s_nvalid - 1);
        const float fl = floorf(r);
        const bool hi_is_lo = ceilf(r) == fl || s_rank + 1 < s_eq;
        const float hi = hi_is_lo ? lo : key_value(s_min_above);
        const float w = r - fl;
        const float d = hi - lo;
        tau[0] = s_nan ? __int_as_float(0x7fffffff) : (fabsf(w) < 0.5f ? __fmaf_rn(w, d, lo) : __fmaf_rn(-d, 1.f - w, hi));
    }
}

}  // namespace

extern "C" {

int br_entropy_threshold(const float* entropy, const int32_t* mask, int64_t n, float level, float* tau, void* stream) {
    BR_CHECK_ARG(n >= 0 && n < (int64_t)UINT32_MAX, "entropy_threshold: n=%lld out of range", (long long)n);
    BR_CHECK_ARG(level >= 0.f && level <= 1.f, "entropy_threshold: level must lie in [0, 1], got %g", (double)level);
    entropy_threshold_kernel<<<1, NT, 0, (cudaStream_t)stream>>>(entropy, mask, (long long)n, level, tau);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // extern "C"
