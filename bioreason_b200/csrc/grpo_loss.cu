// GRPO group-relative advantages and the clipped-ratio + k3-KL loss (forward and analytic backward) --
// single-launch warp-reduction kernels.  Reference: bioreason/trainer/grpo_trainer.py:605-609 (EOS mask),
// :682-692 (advantages), :786-812 (loss, mean_kl, clip_ratio).  SURVEY.md §2.3 K9-K11.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

namespace {

// one warp per group of G consecutive rows
__global__ void advantages_kernel(const float* __restrict__ rpf, int rows, int nf, int G, float* __restrict__ adv,
                                  float* __restrict__ gmean, float* __restrict__ gstd) {
    const int grp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (grp * G >= rows) return;
    const int r0 = grp * G;
    float s = 0.f;
    for (int i = lane; i < G; i += 32) {
        float r = 0.f;
        for (int f = 0; f < nf; ++f) r += rpf[(size_t)(r0 + i) * nf + f];
        s += r;
    }
    const float mean = br::warp_sum(s) / (float)G;
    float v = 0.f;
    for (int i = lane; i < G; i += 32) {
        float r = 0.f;
        for (int f = 0; f < nf; ++f) r += rpf[(size_t)(r0 + i) * nf + f];
        v += (r - mean) * (r - mean);
    }
    const float sd = sqrtf(br::warp_sum(v) / (float)(G - 1));     // torch.std: unbiased
    for (int i = lane; i < G; i += 32) {
        float r = 0.f;
        for (int f = 0; f < nf; ++f) r += rpf[(size_t)(r0 + i) * nf + f];
        adv[r0 + i] = (r - mean) / (sd + 1e-4f);
    }
    if (lane == 0) {
        if (gmean) gmean[grp] = mean;
        if (gstd) gstd[grp] = sd;
    }
}

// one CTA, one warp per row (strided); fixed-order reductions -> deterministic.
// IS: truncated importance sampling against the rollout's own log-probs b = rollout_lp: the policy-gradient term of each token is
// weighted by w = min(exp(o - b), is_cap) with o = old_lp (lp when old_lp is NULL), a value without gradient; the KL term is not
// weighted.  is_stats = masked token means of {w, [exp(o - b) > is_cap], o - b, exp(o - b) - 1 - (o - b)}.
template <bool IS>
__global__ void __launch_bounds__(1024) grpo_loss_kernel(const float* __restrict__ lp, const float* __restrict__ old_lp,
                                                         const float* __restrict__ ref_lp, const float* __restrict__ adv,
                                                         const int* __restrict__ mask, int B, int C, float beta, float eps_lo,
                                                         float eps_hi, float* __restrict__ out3, float* __restrict__ dlp,
                                                         const float* __restrict__ rollout_lp, float is_cap, float* __restrict__ is_stats) {
    __shared__ float s_loss[32], s_kl[32], s_clip[32], s_cnt[32];
    __shared__ float s_is[IS ? 4 : 1][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    float w_loss = 0.f, w_kl = 0.f, w_clip = 0.f, w_cnt = 0.f;
    float w_is[4] = {0.f, 0.f, 0.f, 0.f};
    for (int b = warp; b < B; b += nwarps) {
        float cnt = 0.f;
        for (int t = lane; t < C; t += 32) cnt += (float)mask[(size_t)b * C + t];
        cnt = br::warp_sum(cnt);
        const float a = adv[b];
        const float inv = cnt > 0.f ? 1.f / (cnt * (float)B) : 0.f;
        float rl = 0.f, rk = 0.f, rc = 0.f;
        float ris[4] = {0.f, 0.f, 0.f, 0.f};
        for (int t = lane; t < C; t += 32) {
            const size_t i = (size_t)b * C + t;
            const float x = lp[i];
            const float o = old_lp ? old_lp[i] : x;
            const float c1 = expf(x - o);
            const float c2 = fminf(fmaxf(c1, 1.f - eps_lo), 1.f + eps_hi);
            const float l1 = c1 * a, l2 = c2 * a;
            float l = -fminf(l1, l2);
            float g;
            if (l1 < l2) g = -c1 * a;
            else if (l1 > l2) g = (c1 > 1.f - eps_lo && c1 < 1.f + eps_hi) ? -c1 * a : 0.f;
            else g = (c1 >= 1.f - eps_lo && c1 <= 1.f + eps_hi) ? -c1 * a : -0.5f * c1 * a;
            if constexpr (IS) {
                const float d = o - rollout_lp[i];
                const float r = expf(d);
                const float w = fminf(r, is_cap);
                l *= w; g *= w;
                const float m = (float)mask[i];
                ris[0] += w * m; ris[1] += (r > is_cap ? m : 0.f); ris[2] += d * m; ris[3] += (r - 1.f - d) * m;
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
            rl += l * m; rk += kl * m; rc += (l1 < l2 ? m : 0.f);
            if (dlp) dlp[i] = g * m * inv;
        }
        rl = br::warp_sum(rl); rk = br::warp_sum(rk); rc = br::warp_sum(rc);
        if (cnt > 0.f) { w_loss += rl / cnt; w_kl += rk / cnt; }
        w_clip += rc; w_cnt += cnt;
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) w_is[j] += br::warp_sum(ris[j]);
        }
    }
    if (lane == 0) { s_loss[warp] = w_loss; s_kl[warp] = w_kl; s_clip[warp] = w_clip; s_cnt[warp] = w_cnt; }
    if constexpr (IS) {
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j) s_is[j][warp] = w_is[j];
        }
    }
    __syncthreads();
    if (warp == 0) {
        float a = lane < nwarps ? s_loss[lane] : 0.f, k = lane < nwarps ? s_kl[lane] : 0.f;
        float c = lane < nwarps ? s_clip[lane] : 0.f, n = lane < nwarps ? s_cnt[lane] : 0.f;
        a = br::warp_sum(a); k = br::warp_sum(k); c = br::warp_sum(c); n = br::warp_sum(n);
        if (lane == 0) { out3[0] = a / (float)B; out3[1] = k / (float)B; out3[2] = n > 0.f ? c / n : 0.f; }
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float s = br::warp_sum(lane < nwarps ? s_is[j][lane] : 0.f);
                if (lane == 0) is_stats[j] = n > 0.f ? s / n : 0.f;
            }
        }
    }
}

// grpo_loss_kernel with high-entropy token selection (TRL's top_entropy_quantile, "Beyond the 80/20 Rule"): the policy-gradient term
// (and its gradient) of token i is kept only where ent[i] >= *tau; the KL term, the row normalisation (sum of mask) and the clip ratio
// are not affected.  ent_sum[0] = sum of mask * ent.  A separate kernel rather than a template flag of grpo_loss_kernel: the extra
// parameters alone change that kernel's register allocation.
template <bool IS>
__global__ void __launch_bounds__(1024) grpo_loss_ent_kernel(const float* __restrict__ lp, const float* __restrict__ old_lp,
                                                             const float* __restrict__ ref_lp, const float* __restrict__ adv,
                                                             const int* __restrict__ mask, int B, int C, float beta, float eps_lo,
                                                             float eps_hi, float* __restrict__ out3, float* __restrict__ dlp,
                                                             const float* __restrict__ rollout_lp, float is_cap, float* __restrict__ is_stats,
                                                                 const float* __restrict__ ent, const float* __restrict__ tau,
                                                                 float* __restrict__ ent_sum) {
    __shared__ float s_loss[32], s_kl[32], s_clip[32], s_cnt[32], s_ent[32];
    __shared__ float s_is[IS ? 4 : 1][32];
    const float thr = *tau;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    float w_loss = 0.f, w_kl = 0.f, w_clip = 0.f, w_cnt = 0.f;
    float w_is[4] = {0.f, 0.f, 0.f, 0.f};
    float w_ent = 0.f;
    for (int b = warp; b < B; b += nwarps) {
        float cnt = 0.f;
        for (int t = lane; t < C; t += 32) cnt += (float)mask[(size_t)b * C + t];
        cnt = br::warp_sum(cnt);
        const float a = adv[b];
        const float inv = cnt > 0.f ? 1.f / (cnt * (float)B) : 0.f;
        float rl = 0.f, rk = 0.f, rc = 0.f;
        float ris[4] = {0.f, 0.f, 0.f, 0.f};
        float rent = 0.f;
        for (int t = lane; t < C; t += 32) {
            const size_t i = (size_t)b * C + t;
            const float x = lp[i];
            const float o = old_lp ? old_lp[i] : x;
            const float c1 = expf(x - o);
            const float c2 = fminf(fmaxf(c1, 1.f - eps_lo), 1.f + eps_hi);
            const float l1 = c1 * a, l2 = c2 * a;
            float l = -fminf(l1, l2);
            float g;
            if (l1 < l2) g = -c1 * a;
            else if (l1 > l2) g = (c1 > 1.f - eps_lo && c1 < 1.f + eps_hi) ? -c1 * a : 0.f;
            else g = (c1 >= 1.f - eps_lo && c1 <= 1.f + eps_hi) ? -c1 * a : -0.5f * c1 * a;
            const float h = ent[i];
            const bool keep = h >= thr;
            if constexpr (IS) {
                const float d = o - rollout_lp[i];
                const float r = expf(d);
                const float w = fminf(r, is_cap);
                const float we = keep ? w : 0.f;                        // through the weight: a kept token's arithmetic is grpo_loss_kernel's
                l *= we; g *= we;
                const float m = (float)mask[i];
                ris[0] += w * m; ris[1] += (r > is_cap ? m : 0.f); ris[2] += d * m; ris[3] += (r - 1.f - d) * m;
            }
            if constexpr (!IS) {
                if (!keep) { l = 0.f; g = 0.f; }                        // a select: a kept token's arithmetic is grpo_loss_kernel's
            }
            rent += h * (float)mask[i];
            float kl = 0.f;
            if (beta > 0.f && ref_lp) {
                const float d = ref_lp[i] - x;
                const float e = expf(d);
                kl = e - d - 1.f;
                l += beta * kl;
                g += beta * (1.f - e);
            }
            const float m = (float)mask[i];
            rl += l * m; rk += kl * m; rc += (l1 < l2 ? m : 0.f);
            if (dlp) dlp[i] = g * m * inv;
        }
        rl = br::warp_sum(rl); rk = br::warp_sum(rk); rc = br::warp_sum(rc);
        if (cnt > 0.f) { w_loss += rl / cnt; w_kl += rk / cnt; }
        w_clip += rc; w_cnt += cnt;
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) w_is[j] += br::warp_sum(ris[j]);
        }
        w_ent += br::warp_sum(rent);
    }
    if (lane == 0) { s_loss[warp] = w_loss; s_kl[warp] = w_kl; s_clip[warp] = w_clip; s_cnt[warp] = w_cnt; s_ent[warp] = w_ent; }
    if constexpr (IS) {
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j) s_is[j][warp] = w_is[j];
        }
    }
    __syncthreads();
    if (warp == 0) {
        float a = lane < nwarps ? s_loss[lane] : 0.f, k = lane < nwarps ? s_kl[lane] : 0.f;
        float c = lane < nwarps ? s_clip[lane] : 0.f, n = lane < nwarps ? s_cnt[lane] : 0.f;
        a = br::warp_sum(a); k = br::warp_sum(k); c = br::warp_sum(c); n = br::warp_sum(n);
        if (lane == 0) { out3[0] = a / (float)B; out3[1] = k / (float)B; out3[2] = n > 0.f ? c / n : 0.f; }
        if constexpr (IS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float s = br::warp_sum(lane < nwarps ? s_is[j][lane] : 0.f);
                if (lane == 0) is_stats[j] = n > 0.f ? s / n : 0.f;
            }
        }
        const float se = br::warp_sum(lane < nwarps ? s_ent[lane] : 0.f);
        if (lane == 0) ent_sum[0] = se;
    }
}

__global__ void eos_mask_kernel(const long long* __restrict__ ids, int B, int C, long long eos, int* __restrict__ mask) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= B) return;
    int first = C;                                     // no EOS -> everything kept
    for (int t = lane; t < C; t += 32)
        if (ids[(size_t)b * C + t] == eos) { first = t; break; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    for (int t = lane; t < C; t += 32) mask[(size_t)b * C + t] = (t <= first) ? 1 : 0;
}

}  // namespace

extern "C" {

int br_grpo_advantages(const float* rpf, int rows, int n_funcs, int G, float* adv, float* gmean, float* gstd, void* stream) {
    BR_CHECK_ARG(rows > 0 && G > 1 && rows % G == 0 && n_funcs > 0, "grpo_advantages: rows=%d must be a positive multiple of G=%d (>1)", rows, G);
    const int groups = rows / G, wpb = 4;
    advantages_kernel<<<(groups + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>(rpf, rows, n_funcs, G, adv, gmean, gstd);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_grpo_loss_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* adv, const int32_t* mask, int B, int C,
                         float beta, float eps_low, float eps_high, float* out3, float* dlp, void* stream) {
    BR_CHECK_ARG(B > 0 && C > 0, "grpo_loss: empty batch");
    BR_CHECK_ARG(!(beta > 0.f && !ref_lp), "grpo_loss: beta > 0 needs ref_lp");
    int threads = B >= 32 ? 1024 : B * 32;
    grpo_loss_kernel<false><<<1, threads, 0, (cudaStream_t)stream>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high, out3, dlp,
                                                                     nullptr, 0.f, nullptr);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_grpo_loss_is_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* rollout_lp, const float* adv,
                            const int32_t* mask, int B, int C, float beta, float eps_low, float eps_high, float is_cap, float* out3,
                            float* is_stats, float* dlp, void* stream) {
    BR_CHECK_ARG(B > 0 && C > 0, "grpo_loss_is: empty batch");
    BR_CHECK_ARG(!(beta > 0.f && !ref_lp), "grpo_loss_is: beta > 0 needs ref_lp");
    BR_CHECK_ARG(rollout_lp && is_stats, "grpo_loss_is: needs rollout_lp and is_stats");
    BR_CHECK_ARG(is_cap > 0.f, "grpo_loss_is: is_cap must be > 0 (+inf: untruncated), got %g", (double)is_cap);
    int threads = B >= 32 ? 1024 : B * 32;
    grpo_loss_kernel<true><<<1, threads, 0, (cudaStream_t)stream>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high, out3, dlp,
                                                                    rollout_lp, is_cap, is_stats);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_grpo_loss_ent_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* rollout_lp, const float* adv,
                             const int32_t* mask, const float* entropy, const float* tau, int B, int C, float beta, float eps_low,
                             float eps_high, float is_cap, float* out3, float* is_stats, float* ent_sum, float* dlp, void* stream) {
    BR_CHECK_ARG(B > 0 && C > 0, "grpo_loss_ent: empty batch");
    BR_CHECK_ARG(!(beta > 0.f && !ref_lp), "grpo_loss_ent: beta > 0 needs ref_lp");
    BR_CHECK_ARG(entropy && tau && ent_sum, "grpo_loss_ent: needs entropy, tau and ent_sum");
    int threads = B >= 32 ? 1024 : B * 32;
    if (rollout_lp) {
        BR_CHECK_ARG(is_stats, "grpo_loss_ent: rollout_lp needs is_stats");
        BR_CHECK_ARG(is_cap > 0.f, "grpo_loss_ent: is_cap must be > 0 (+inf: untruncated), got %g", (double)is_cap);
        grpo_loss_ent_kernel<true><<<1, threads, 0, (cudaStream_t)stream>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high,
                                                                            out3, dlp, rollout_lp, is_cap, is_stats, entropy, tau, ent_sum);
    } else {
        grpo_loss_ent_kernel<false><<<1, threads, 0, (cudaStream_t)stream>>>(lp, old_lp, ref_lp, adv, mask, B, C, beta, eps_low, eps_high,
                                                                             out3, dlp, nullptr, 0.f, nullptr, entropy, tau, ent_sum);
    }
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_eos_mask(const int64_t* ids, int B, int C, int64_t eos_id, int32_t* mask, void* stream) {
    BR_CHECK_ARG(B > 0 && C > 0, "eos_mask: empty");
    const int wpb = 4;
    eos_mask_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>((const long long*)ids, B, C, (long long)eos_id, mask);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // extern "C"
