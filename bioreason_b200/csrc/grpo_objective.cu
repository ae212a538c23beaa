// The GRPO objectives of later TRL releases: loss_type (grpo / bnpo / dr_grpo / dapo), sequence-level importance ratios (GSPO),
// two-sided clipping (delta), advantage scaling (scale_rewards) and the completion mask of mask_truncated_completions.  The
// contract is DESIGN.md §3; the kernels of grpo_loss.cu stay as they are and remain the default path.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

#include <math.h>

namespace {

constexpr int OUT_N = 7;      // {loss, sum of row-mean kl, clip, low, high, region, tokens}

// d(-min(q a, c2 a)) / ds for coef_1 = c1 = exp(s), q = min(c1, delta) (torch.clamp(max=delta): passes at the bound),
// c2 = clamp(c1, 1 - eps_lo, 1 + eps_hi) (passes at the bounds); torch.min splits the gradient evenly at a tie.  Without delta
// (pd true) every branch is grpo_loss_kernel's arithmetic.
__device__ __forceinline__ float clip_grad(float c1, float a, float l1, float l2, bool pd, float eps_lo, float eps_hi) {
    const bool pc = c1 >= 1.f - eps_lo && c1 <= 1.f + eps_hi;
    if (l1 < l2) return pd ? -c1 * a : 0.f;
    if (l1 > l2) return pc ? -c1 * a : 0.f;
    if (pd && pc) return -c1 * a;
    return (pd || pc) ? -0.5f * c1 * a : 0.f;
}

// One CTA, one warp per row (strided), fixed-order reductions: deterministic, no atomics.  The structure and the arithmetic of a
// token at the defaults (token level, no delta, norm_rows = B) are grpo_loss_kernel's / grpo_loss_ent_kernel's, so those outputs
// come out bit for bit.  At sequence level a first pass over the row gives |o_b| = sum m, sum m (lp - o) and W_b = sum m w k.
template <bool IS, bool ENT>
__global__ void __launch_bounds__(1024) grpo_objective_kernel(const float* __restrict__ lp, const float* __restrict__ old_lp,
                                                              const float* __restrict__ ref_lp, const float* __restrict__ adv,
                                                              const int* __restrict__ mask, int B, int C, float beta, float eps_lo,
                                                              float eps_hi, br_grpo_objective opt, float* __restrict__ out,
                                                              float* __restrict__ dlp) {
    __shared__ float s_out[OUT_N][32];
    __shared__ float s_is[IS ? 4 : 1][32];
    __shared__ float s_ent[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const bool seq = opt.sequence_level != 0;
    const bool has_delta = opt.delta < INFINITY;
    const float delta = opt.delta;
    const bool rows_norm = opt.norm_rows > 0;
    const float D = rows_norm ? (float)opt.norm_rows : *opt.norm;
    const float* __restrict__ rollout_lp = opt.rollout_lp;
    const float is_cap = opt.is_cap;
    const float* __restrict__ ent = opt.entropy;
    const float thr = ENT ? *opt.tau : 0.f;
    float w_out[OUT_N];
#pragma unroll
    for (int j = 0; j < OUT_N; ++j) w_out[j] = 0.f;
    float w_is[4] = {0.f, 0.f, 0.f, 0.f};
    float w_ent = 0.f;
    for (int b = warp; b < B; b += nwarps) {
        float cnt = 0.f, sdiff = 0.f, sw = 0.f;
        for (int t = lane; t < C; t += 32) {
            const size_t i = (size_t)b * C + t;
            const float m = (float)mask[i];
            cnt += m;
            if (seq) {
                const float x = lp[i];
                const float o = old_lp ? old_lp[i] : x;
                sdiff += (x - o) * m;
                float w = 1.f;
                if constexpr (IS) w = fminf(expf(o - rollout_lp[i]), is_cap);
                if constexpr (ENT) w = ent[i] >= thr ? w : 0.f;
                sw += w * m;
            }
        }
        cnt = br::warp_sum(cnt);
        const float a = adv[b];
        const float inv = rows_norm ? (cnt > 0.f ? 1.f / (cnt * D) : 0.f) : 1.f / D;
        float c1_row = 1.f, g_row = 0.f;
        if (seq) {
            const float nrm = fmaxf(cnt, 1.f);
            c1_row = expf(br::warp_sum(sdiff) / nrm);
            const float c2 = fminf(fmaxf(c1_row, 1.f - eps_lo), 1.f + eps_hi);
            const float q = has_delta ? fminf(c1_row, delta) : c1_row;
            const float g = clip_grad(c1_row, a, q * a, c2 * a, !has_delta || c1_row <= delta, eps_lo, eps_hi);
            g_row = g * (br::warp_sum(sw) / nrm);               // d/dlp_t of sum_t' m w k (-min) = g W_b m_t / |o_b|
        }
        float rl = 0.f, rk = 0.f, rc = 0.f, rlo = 0.f, rhi = 0.f, rreg = 0.f;
        float ris[4] = {0.f, 0.f, 0.f, 0.f};
        float rent = 0.f;
        for (int t = lane; t < C; t += 32) {
            const size_t i = (size_t)b * C + t;
            const float x = lp[i];
            const float o = old_lp ? old_lp[i] : x;
            const float c1 = seq ? c1_row : expf(x - o);
            const float c2 = fminf(fmaxf(c1, 1.f - eps_lo), 1.f + eps_hi);
            const float q = has_delta ? fminf(c1, delta) : c1;
            const float l1 = q * a, l2 = c2 * a;
            float l = -fminf(l1, l2);
            float g = seq ? 0.f : clip_grad(c1, a, l1, l2, !has_delta || c1 <= delta, eps_lo, eps_hi);
            bool keep = true;
            if constexpr (ENT) {
                const float h = ent[i];
                keep = h >= thr;
                rent += h * (float)mask[i];
            }
            if constexpr (IS) {
                const float d = o - rollout_lp[i];
                const float r = expf(d);
                const float w = fminf(r, is_cap);
                const float we = keep ? w : 0.f;
                l *= we; g *= we;
                const float m = (float)mask[i];
                ris[0] += w * m; ris[1] += (r > is_cap ? m : 0.f); ris[2] += d * m; ris[3] += (r - 1.f - d) * m;
            }
            if constexpr (ENT && !IS) {
                if (!keep) { l = 0.f; g = 0.f; }
            }
            float kl = 0.f;
            if (beta > 0.f && ref_lp) {
                const float d = ref_lp[i] - x;
                const float e = expf(d);
                kl = e - d - 1.f;
                l += beta * kl;
                g += beta * (1.f - e);
            }
            const float m = (float)mask[i];
            const bool low = q < 1.f - eps_lo && a < 0.f, high = q > 1.f + eps_hi && a > 0.f;
            rl += l * m; rk += kl * m; rc += (l1 < l2 ? m : 0.f);
            rlo += low ? m : 0.f; rhi += high ? m : 0.f; rreg += (low || high) ? m : 0.f;
            if (dlp) dlp[i] = seq ? (g_row + g) * m * inv : g * m * inv;
        }
        rl = br::warp_sum(rl); rk = br::warp_sum(rk); rc = br::warp_sum(rc);
        if (rows_norm) {
            if (cnt > 0.f) w_out[0] += rl / cnt;
        } else {
            w_out[0] += rl;
        }
        if (cnt > 0.f) w_out[1] += rk / cnt;
        w_out[2] += rc;
        w_out[3] += br::warp_sum(rlo); w_out[4] += br::warp_sum(rhi); w_out[5] += br::warp_sum(rreg);
        w_out[6] += cnt;
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) w_is[j] += br::warp_sum(ris[j]);
        }
        if constexpr (ENT) w_ent += br::warp_sum(rent);
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < OUT_N; ++j) s_out[j][warp] = w_out[j];
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) s_is[j][warp] = w_is[j];
        }
        s_ent[warp] = w_ent;
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int j = 0; j < OUT_N; ++j) {
            const float s = br::warp_sum(lane < nwarps ? s_out[j][lane] : 0.f);
            if (lane == 0) out[j] = j == 0 ? s / D : s;
        }
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float s = br::warp_sum(lane < nwarps ? s_is[j][lane] : 0.f);
                if (lane == 0) opt.is_sums[j] = s;
            }
        }
        if constexpr (ENT) {
            const float s = br::warp_sum(lane < nwarps ? s_ent[lane] : 0.f);
            if (lane == 0) opt.ent_sum[0] = s;
        }
    }
}

__device__ __forceinline__ float row_reward(const float* __restrict__ rpf, int row, int nf) {
    float r = 0.f;
    for (int f = 0; f < nf; ++f) r += rpf[(size_t)row * nf + f];
    return r;
}

// fixed-order sum over the CTA; every thread gets the result
__device__ float block_sum(float v, float* s_red) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    v = br::warp_sum(v);
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    return br::warp_sum(lane < nwarps ? s_red[lane] : 0.f);
}

// One CTA.  Group statistics: one warp per group of G consecutive rows (strided), advantages_kernel's arithmetic.  Batch mode: one
// std over all rows, two passes (mean, then the sum of squared deviations), unbiased.  std_used[row] is the std the row's advantage
// divides by (the group std in "none" mode, which divides by nothing); zero_std[row] = std_used <= 1e-8.
__global__ void __launch_bounds__(1024) advantages_scaled_kernel(const float* __restrict__ rpf, int rows, int nf, int G, int mode,
                                                                 float* __restrict__ adv, float* __restrict__ std_used,
                                                                 int32_t* __restrict__ zero_std) {
    __shared__ float s_red[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    float bstd = 0.f;
    if (mode == BR_SCALE_REWARDS_BATCH) {
        float s = 0.f;
        for (int i = threadIdx.x; i < rows; i += blockDim.x) s += row_reward(rpf, i, nf);
        const float mean = block_sum(s, s_red) / (float)rows;
        float v = 0.f;
        for (int i = threadIdx.x; i < rows; i += blockDim.x) {
            const float d = row_reward(rpf, i, nf) - mean;
            v += d * d;
        }
        bstd = sqrtf(block_sum(v, s_red) / (float)(rows - 1));
    }
    for (int grp = warp; grp * G < rows; grp += nwarps) {
        const int r0 = grp * G;
        float s = 0.f;
        for (int i = lane; i < G; i += 32) s += row_reward(rpf, r0 + i, nf);
        const float mean = br::warp_sum(s) / (float)G;
        float v = 0.f;
        for (int i = lane; i < G; i += 32) {
            const float r = row_reward(rpf, r0 + i, nf);
            v += (r - mean) * (r - mean);
        }
        const float sd = mode == BR_SCALE_REWARDS_BATCH ? bstd : sqrtf(br::warp_sum(v) / (float)(G - 1));
        for (int i = lane; i < G; i += 32) {
            const float r = row_reward(rpf, r0 + i, nf);
            adv[r0 + i] = mode == BR_SCALE_REWARDS_NONE ? r - mean : (r - mean) / (sd + 1e-4f);
            std_used[r0 + i] = sd;
            zero_std[r0 + i] = sd <= 1e-8f ? 1 : 0;
        }
    }
}

// eos_mask_kernel with the rows that hold no EOS zeroed; lengths[b] = the row's mask count before that (min(first EOS + 1, C))
__global__ void eos_mask_truncated_kernel(const long long* __restrict__ ids, int B, int C, long long eos, int* __restrict__ mask,
                                          int* __restrict__ lengths) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= B) return;
    int first = C;
    for (int t = lane; t < C; t += 32)
        if (ids[(size_t)b * C + t] == eos) { first = t; break; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    const bool truncated = first == C;
    for (int t = lane; t < C; t += 32) mask[(size_t)b * C + t] = (!truncated && t <= first) ? 1 : 0;
    if (lane == 0) lengths[b] = min(first + 1, C);
}

}  // namespace

extern "C" {

int br_grpo_objective_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* adv, const int32_t* mask, int B,
                              int C, float beta, float eps_low, float eps_high, const br_grpo_objective* opt, float* out7, float* dlp,
                              void* stream) {
    BR_CHECK_ARG(B > 0 && C > 0, "grpo_objective: empty batch");
    BR_CHECK_ARG(opt && out7, "grpo_objective: needs opt and out7");
    BR_CHECK_ARG(!(beta > 0.f && !ref_lp), "grpo_objective: beta > 0 needs ref_lp");
    BR_CHECK_ARG(opt->norm_rows > 0 || (opt->norm_rows == 0 && opt->norm), "grpo_objective: needs norm_rows > 0 or a device norm");
    BR_CHECK_ARG(opt->delta > 0.f, "grpo_objective: delta must be > 0 (+inf: off), got %g", (double)opt->delta);
    if (opt->rollout_lp) {
        BR_CHECK_ARG(opt->is_sums, "grpo_objective: rollout_lp needs is_sums");
        BR_CHECK_ARG(opt->is_cap > 0.f, "grpo_objective: is_cap must be > 0 (+inf: untruncated), got %g", (double)opt->is_cap);
    }
    if (opt->entropy) BR_CHECK_ARG(opt->tau && opt->ent_sum, "grpo_objective: entropy needs tau and ent_sum");
    const int threads = B >= 32 ? 1024 : B * 32;
    cudaStream_t st = (cudaStream_t)stream;
    if (opt->rollout_lp && opt->entropy)
        grpo_objective_kernel<true, true><<<1, threads, 0, st>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high, *opt, out7, dlp);
    else if (opt->rollout_lp)
        grpo_objective_kernel<true, false><<<1, threads, 0, st>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high, *opt, out7, dlp);
    else if (opt->entropy)
        grpo_objective_kernel<false, true><<<1, threads, 0, st>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high, *opt, out7, dlp);
    else
        grpo_objective_kernel<false, false><<<1, threads, 0, st>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high, *opt, out7, dlp);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_grpo_advantages_scaled(const float* rpf, int rows, int n_funcs, int G, int mode, float* adv, float* std_used, int32_t* zero_std,
                              void* stream) {
    BR_CHECK_ARG(rows > 0 && G > 1 && rows % G == 0 && n_funcs > 0, "grpo_advantages_scaled: rows=%d must be a positive multiple of G=%d (>1)",
                 rows, G);
    BR_CHECK_ARG(mode == BR_SCALE_REWARDS_GROUP || mode == BR_SCALE_REWARDS_BATCH || mode == BR_SCALE_REWARDS_NONE,
                 "grpo_advantages_scaled: unknown mode %d", mode);
    BR_CHECK_ARG(adv && std_used && zero_std, "grpo_advantages_scaled: needs adv, std_used and zero_std");
    const int groups = rows / G;
    const int threads = groups >= 32 || mode == BR_SCALE_REWARDS_BATCH ? 1024 : groups * 32;
    advantages_scaled_kernel<<<1, threads, 0, (cudaStream_t)stream>>>(rpf, rows, n_funcs, G, mode, adv, std_used, zero_std);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_eos_mask_truncated(const int64_t* ids, int B, int C, int64_t eos_id, int32_t* mask, int32_t* lengths, void* stream) {
    BR_CHECK_ARG(B > 0 && C > 0, "eos_mask_truncated: empty");
    BR_CHECK_ARG(mask && lengths, "eos_mask_truncated: needs mask and lengths");
    const int wpb = 4;
    eos_mask_truncated_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>((const long long*)ids, B, C, (long long)eos_id,
                                                                                           mask, lengths);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // extern "C"
