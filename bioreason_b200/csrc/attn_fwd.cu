// C entry points of the flash-attention forward (br_attn_fwd, br_attn_fwd_shared): argument checks + dispatch to the wgmma / TMA kernel in
// attn_fwd_tc5.cu.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

int br_attn_fwd_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo, float* lse,
                         int B, int L, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* kv_start, const int32_t* kv_end,
                         float scale, int causal, cudaStream_t st);
int br_attn_fwd_shared_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                                float* lse_prefix, float* lse_suffix, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads,
                                const int32_t* kv_start, const int32_t* kv_end, float scale, cudaStream_t st);

extern "C" int br_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo, float* lse,
                           int B, int L, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* kv_start, const int32_t* kv_end,
                           float scale, int causal, void* stream) {
    BR_CHECK_ARG(B > 0 && L > 0 && n_q_heads % n_kv_heads == 0, "attn_fwd: bad shape B=%d L=%d Hq=%d Hkv=%d", B, L, n_q_heads, n_kv_heads);
    BR_CHECK_ARG(head_dim == 128 || head_dim == 64, "attn_fwd: head_dim must be 64 or 128");
    BR_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "attn_fwd: strides must be multiples of 8 elements");
    return br_attn_fwd_tc5_impl(q, ldq, k, ldk, v, ldv, o, ldo, lse, B, L, n_q_heads, n_kv_heads, head_dim, kv_start, kv_end, scale, causal,
                                (cudaStream_t)stream);
}

extern "C" int br_attn_fwd_shared(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                                  float* lse_prefix, float* lse_suffix, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads,
                                  int head_dim, const int32_t* kv_start, const int32_t* kv_end, float scale, void* stream) {
    BR_CHECK_ARG(U > 0 && G > 0 && Lp >= 0 && Lp % 64 == 0 && Ls > 0 && n_q_heads % n_kv_heads == 0,
                 "attn_fwd_shared: bad shape U=%d G=%d Lp=%d Ls=%d Hq=%d Hkv=%d", U, G, Lp, Ls, n_q_heads, n_kv_heads);
    BR_CHECK_ARG(head_dim == 128, "attn_fwd_shared: head_dim 128 (the decoder) only");
    BR_CHECK_ARG(kv_start && kv_end && lse_suffix && (Lp == 0 || lse_prefix), "attn_fwd_shared: kv_start, kv_end and both lse buffers are required");
    BR_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "attn_fwd_shared: strides must be multiples of 8 elements");
    return br_attn_fwd_shared_tc5_impl(q, ldq, k, ldk, v, ldv, o, ldo, lse_prefix, lse_suffix, U, G, Lp, Ls, n_q_heads, n_kv_heads, kv_start,
                                       kv_end, scale, (cudaStream_t)stream);
}
