// Pooled score head of a sequence-classification reward model (HF GenericForSequenceClassification on Qwen3, transformers 5.5
// modeling_layers.py): per row b of a right- or left-padded batch
//   t_b   = the rightmost column whose id is not pad_id (argmax over zeros -> 0 when every column is pad; no pad id -> L - 1)
//   y     = bf16(w_norm * bf16(h[b, t_b] * rsqrt(mean(h^2) + eps)))          (Qwen3RMSNorm, fp32 sum of squares)
//   out_j = float(bf16(sum_i y_i S[j, i]))                                    (bf16 Linear: fp32 accumulation, bf16 output)
// h is the last decoder layer's output before the final norm, so only the pooled row is normed and scored.
// One CTA per row, fixed-order reductions (per-thread strided sums -> xor-shuffle warp sums -> warp partials added in warp order by
// one thread): no atomics, the same bits on every launch.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

namespace {

constexpr int NT = 256;
constexpr int NW = NT / 32;
constexpr int MAX_D = 10240;

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16(x)); }

// fixed-order block sum; every thread gets the total
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = br::warp_sum(v);
    __syncthreads();                                       // red[] may still be read by the previous call
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) s += red[w];
    return s;
}

__global__ void __launch_bounds__(NT) seqcls_score_kernel(const bf16* __restrict__ h, long long ldh, const long long* __restrict__ ids,
                                                          int L, long long pad_id, const bf16* __restrict__ norm_w, float eps,
                                                          const bf16* __restrict__ score_w, long long ldw, int n_labels, int d,
                                                          float* __restrict__ out, long long ldo, int* __restrict__ index) {
    __shared__ __align__(16) bf16 y[MAX_D];
    __shared__ float red[NW];
    __shared__ int s_idx[NW];
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    // pooled position: the rightmost non-pad column (max is order-independent)
    int t = -1;
    if (pad_id < 0) {
        t = L - 1;
    } else {
        const long long* row_ids = ids + (long long)b * L;
        for (int c = threadIdx.x; c < L; c += NT)
            if (row_ids[c] != pad_id) t = c;               // c grows along the loop: the last hit is this thread's largest
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t = max(t, __shfl_xor_sync(0xffffffffu, t, o));
        if (lane == 0) s_idx[warp] = t;
        __syncthreads();
#pragma unroll
        for (int w = 0; w < NW; ++w) t = max(t, s_idx[w]);
        if (t < 0) t = 0;                                  // all pad: argmax of zeros
    }
    if (index != nullptr && threadIdx.x == 0) index[b] = t;

    // final RMSNorm of the pooled row, HF's rounding points
    const uint4* xp = reinterpret_cast<const uint4*>(h + ((long long)b * L + t) * ldh);
    const uint4* wp = reinterpret_cast<const uint4*>(norm_w);
    const int nvec = d >> 3;
    float ss = 0.f;
    for (int i = threadIdx.x; i < nvec; i += NT) {
        const uint4 v = xp[i];
        const float2 a = br::unpack_bf16(v.x), c = br::unpack_bf16(v.y), e = br::unpack_bf16(v.z), f = br::unpack_bf16(v.w);
        ss += a.x * a.x + a.y * a.y + c.x * c.x + c.y * c.y + e.x * e.x + e.y * e.y + f.x * f.x + f.y * f.y;
    }
    const float rstd = rsqrtf(block_sum(ss, red) / (float)d + eps);
    uint4* yp = reinterpret_cast<uint4*>(y);
    for (int i = threadIdx.x; i < nvec; i += NT) {
        const uint4 v = xp[i], g = wp[i];
        const uint32_t xs[4] = {v.x, v.y, v.z, v.w}, gs[4] = {g.x, g.y, g.z, g.w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 xv = br::unpack_bf16(xs[k]), gv = br::unpack_bf16(gs[k]);
            o[k] = br::pack_bf16(gv.x * rbf(xv.x * rstd), gv.y * rbf(xv.y * rstd));
        }
        yp[i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
    __syncthreads();

    // score rows: fp32 dot products, rounded to bf16 like the Linear's output
    for (int j = 0; j < n_labels; ++j) {
        const uint4* sp = reinterpret_cast<const uint4*>(score_w + (long long)j * ldw);
        float acc = 0.f;
        for (int i = threadIdx.x; i < nvec; i += NT) {
            const uint4 v = yp[i], s = sp[i];
            const uint32_t ys[4] = {v.x, v.y, v.z, v.w}, sw[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 a = br::unpack_bf16(ys[k]), c = br::unpack_bf16(sw[k]);
                acc = fmaf(a.x, c.x, acc);
                acc = fmaf(a.y, c.y, acc);
            }
        }
        const float tot = block_sum(acc, red);
        if (threadIdx.x == 0) out[(long long)b * ldo + j] = rbf(tot);
    }
}

}  // namespace

extern "C" {

int br_seqcls_score(const void* h, int64_t ldh, const int64_t* input_ids, int B, int L, int64_t pad_id, const void* norm_w, float eps,
                    const void* score_w, int64_t ldw, int n_labels, int d, float* out, int64_t ldo, int32_t* index, void* stream) {
    BR_CHECK_ARG(B > 0 && L > 0 && n_labels > 0, "seqcls_score: bad shape B=%d L=%d n_labels=%d", B, L, n_labels);
    BR_CHECK_ARG(d > 0 && d % 8 == 0 && d <= MAX_D, "seqcls_score: d=%d must be a multiple of 8, <= %d", d, MAX_D);
    BR_CHECK_ARG(ldh % 8 == 0 && ldh >= d && ldw % 8 == 0 && ldw >= d && ldo >= n_labels, "seqcls_score: bad strides ldh=%lld ldw=%lld ldo=%lld",
                 (long long)ldh, (long long)ldw, (long long)ldo);
    BR_CHECK_ARG(pad_id >= -1, "seqcls_score: pad_id=%lld (-1: none)", (long long)pad_id);
    BR_CHECK_ARG(h && input_ids && norm_w && score_w && out, "seqcls_score: null argument");
    BR_CHECK_ARG((uintptr_t)h % 16 == 0 && (uintptr_t)norm_w % 16 == 0 && (uintptr_t)score_w % 16 == 0, "seqcls_score: h, norm_w, score_w must be 16-byte aligned");
    seqcls_score_kernel<<<B, NT, 0, (cudaStream_t)stream>>>((const bf16*)h, (long long)ldh, (const long long*)input_ids, L, (long long)pad_id,
                                                           (const bf16*)norm_w, eps, (const bf16*)score_w, (long long)ldw, n_labels, d, out,
                                                           (long long)ldo, index);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // extern "C"
