// C entry points of the flash-attention backward (br_attn_bwd, br_attn_bwd_shared and their workspace sizes): argument checks + dispatch to the two
// deterministic wgmma kernels in attn_bwd_tc5.cu.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

int br_attn_bwd_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                         const void* dout, int64_t lddo, const float* lse, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv,
                         int B, int L, int n_q_heads, int n_kv_heads, const int32_t* kv_start, const int32_t* kv_end, float scale,
                         void* workspace, cudaStream_t st);
int64_t br_attn_bwd_shared_workspace_bytes_impl(int U, int G, int Lp, int Ls, int n_q_heads);
int br_attn_bwd_shared_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                                const void* dout, int64_t lddo, const float* lse_prefix, const float* lse_suffix, void* dq, int64_t lddq,
                                void* dk, int64_t lddk, void* dv, int64_t lddv, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads,
                                const int32_t* kv_start, const int32_t* kv_end, float scale, void* workspace, cudaStream_t st);

extern "C" {

/* delta = rowsum(dO o O): [B, Hq, L] fp32 -- the only workspace the backward needs */
int64_t br_attn_bwd_workspace_bytes(int B, int L, int n_q_heads, int head_dim) {
    (void)head_dim;
    return (int64_t)B * L * n_q_heads * sizeof(float);
}

int br_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo, const void* dout,
                int64_t lddo, const float* lse, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int B, int L, int n_q_heads,
                int n_kv_heads, int head_dim, const int32_t* kv_start, const int32_t* kv_end, float scale, void* workspace, void* stream) {
    BR_CHECK_ARG(head_dim == 128, "attn_bwd: head_dim 128 (the decoder) only; the encoder is forward-only (dna_llm.py:121)");
    BR_CHECK_ARG(B > 0 && L > 0 && n_q_heads % n_kv_heads == 0 && workspace, "attn_bwd: bad shape / missing workspace");
    return br_attn_bwd_tc5_impl(q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse, dq, lddq, dk, lddk, dv, lddv, B, L, n_q_heads, n_kv_heads,
                                kv_start, kv_end, scale, workspace, (cudaStream_t)stream);
}

/* delta of the prefix and suffix queries, then the suffix-coordinate windows */
int64_t br_attn_bwd_shared_workspace_bytes(int U, int G, int Lp, int Ls, int n_q_heads, int head_dim) {
    (void)head_dim;
    return br_attn_bwd_shared_workspace_bytes_impl(U, G, Lp, Ls, n_q_heads);
}

int br_attn_bwd_shared(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                       const void* dout, int64_t lddo, const float* lse_prefix, const float* lse_suffix, void* dq, int64_t lddq, void* dk,
                       int64_t lddk, void* dv, int64_t lddv, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads, int head_dim,
                       const int32_t* kv_start, const int32_t* kv_end, float scale, void* workspace, void* stream) {
    BR_CHECK_ARG(head_dim == 128, "attn_bwd_shared: head_dim 128 (the decoder) only");
    BR_CHECK_ARG(U > 0 && G > 0 && Lp >= 0 && Lp % 64 == 0 && Ls > 0 && n_q_heads % n_kv_heads == 0 && workspace,
                 "attn_bwd_shared: bad shape U=%d G=%d Lp=%d Ls=%d / missing workspace", U, G, Lp, Ls);
    BR_CHECK_ARG(kv_start && kv_end && lse_suffix && (Lp == 0 || lse_prefix), "attn_bwd_shared: kv_start, kv_end and both lse buffers are required");
    return br_attn_bwd_shared_tc5_impl(q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse_prefix, lse_suffix, dq, lddq, dk, lddk, dv, lddv, U, G, Lp,
                                       Ls, n_q_heads, n_kv_heads, kv_start, kv_end, scale, workspace, (cudaStream_t)stream);
}

}  // extern "C"
