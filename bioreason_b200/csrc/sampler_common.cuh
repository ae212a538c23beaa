// Helpers shared by the rollout samplers (sampler.cu: top-k <= 1024; sampler_full.cu: the full vocabulary): the order-preserving key
// of an fp32 logit, HF's logits processors as the kernels apply them, and the fixed-order block reductions.
#pragma once
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

namespace {

__device__ __forceinline__ uint32_t fkey(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float block_max(float v, float* s_red) {   // all threads get the maximum; s_red: 32 floats
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float m = lane < nw ? s_red[lane] : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __syncthreads();
    return m;
}
// fixed-order block sum: thread 0 gets the total (the same bits on every call); s_red: 32 floats
__device__ __forceinline__ float block_sum(float v, float* s_red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = br::warp_sum(v);
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float s = lane < nw ? s_red[lane] : 0.f;
    s = br::warp_sum(s);
    __syncthreads();
    return s;
}

// Processed path (the *_proc entry points, PROC = true): HF's RepetitionPenalty -> MinNewTokens logits processors ahead of temperature /
// top-k / top-p, and MinP after top-p.  Every kernel that reads a logit of the row applies proc_logit to it (stage 1 to the 16 values it
// holds in registers, stage 2 and the single-stage sampler wherever they select on the row itself), so the candidates carry processed
// values.  The log-prob stays on the raw row.  presence[r] is a bitmap of the tokens row r has emitted (bit j of word j / 32); the
// sampler sets the emitted token's bit after the draw, one writer per row.
struct Proc {
    uint32_t* presence;           // [R, ceil(V / 32)], or nullptr: no penalty and no update
    float theta;                  // repetition penalty
    float min_p;                  // 0: off
    int min_new;                  // EOS gets -inf while *step < min_new
    long long eos;                // < 0: no EOS
    const int* step;              // nullptr: step 0
};

// HF RepetitionPenaltyLogitsProcessor (z < 0 ? z * theta : z / theta, fp32, IEEE division) then MinNewTokensLengthLogitsProcessor
__device__ __forceinline__ float proc_logit(float z, bool in_set, bool blocked, float theta) {
    if (in_set) z = z < 0.f ? __fmul_rn(z, theta) : __fdiv_rn(z, theta);
    return blocked ? -INFINITY : z;
}
__device__ __forceinline__ bool proc_in_set(const uint32_t* pres, int id) {
    return pres != nullptr && ((__ldcg(pres + (id >> 5)) >> (id & 31)) & 1u);
}

}  // namespace

// the processed entry points' arguments as the kernels take them; refuses what HF's processors refuse
static int proc_args(const br_sample_proc* proc, int64_t eos_id, const int32_t* step, const char* what, Proc* out) {
    BR_CHECK_ARG(proc, "%s: no br_sample_proc", what);
    BR_CHECK_ARG(proc->repetition_penalty > 0.f, "%s: repetition_penalty must be > 0", what);
    BR_CHECK_ARG(proc->min_p >= 0.f && proc->min_p <= 1.f, "%s: min_p must be in [0, 1]", what);
    BR_CHECK_ARG(proc->min_new_tokens >= 0, "%s: min_new_tokens must be >= 0", what);
    BR_CHECK_ARG(proc->repetition_penalty == 1.f || proc->presence, "%s: repetition_penalty != 1 needs a presence bitmap", what);
    *out = Proc{proc->presence, proc->repetition_penalty, proc->min_p, proc->min_new_tokens, (long long)eos_id, step};
    return BR_OK;
}
