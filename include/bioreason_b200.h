/* libbioreason_b200 -- C ABI of the sm_90a (H100) BioReason hot path.
 *
 * The reference (bowang-lab/BioReason) has no FFI: its hot path is Python calling HuggingFace/PyTorch
 * (SURVEY.md §8b).  This header is the boundary the build introduces *below* the reference's Python
 * surface (`DNALLMModel`, `DNALLMGRPOTrainer`); each entry point names the reference call site it
 * replaces.  Conventions:
 *   - plain pointers + sizes, no torch types; every pointer is a CUDA device pointer unless noted;
 *   - every call enqueues on `stream` (a cudaStream_t) and returns without synchronising;
 *   - return 0 on success, <0 on error; `br_last_error()` gives the (thread-local) message;
 *   - the caller (PyTorch) owns all buffers (including every workspace / scratch buffer named below); the library keeps no
 *     pointer past the call.  There is no communicator handle: the two collectives of the path (reward all-gather, flat
 *     gradient all-reduce; SURVEY.md §8e) are issued by the host through torch.distributed / NCCL, not through this ABI;
 *   - tensors are (pointer, leading dimension in elements) pairs, row-major; there is no tensor struct;
 *   - bf16 = __nv_bfloat16 storage, fp32 accumulation everywhere.
 * This file is parsed by cffi (ABI mode): keep it plain C, no macros beyond the constants below.
 */
#ifndef BIOREASON_B200_H
#define BIOREASON_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BR_BF16 0
#define BR_F32 1

int br_version(void);
/* copies the calling thread's last error message into buf (NUL-terminated); returns its length */
int br_last_error(char* buf, size_t n);
/* 1 if the visible device is sm_90 (H100); the library refuses to run elsewhere */
int br_device_ok(void);

/* ---------------------------------------------------------------------------------------------
 * GRPO advantages + loss  (replaces bioreason/trainer/grpo_trainer.py:682-692 and :786-812)
 * ------------------------------------------------------------------------------------------- */
/* rewards_per_func [rows, n_funcs] f32 -> advantages [rows] f32; groups are G consecutive rows. */
int br_grpo_advantages(const float* rewards_per_func, int rows, int n_funcs, int G, float* advantages,
                       float* group_mean, float* group_std, void* stream);
/* lp/old_lp/ref_lp [B, C] f32 (old_lp NULL => mu == 1; ref_lp NULL => beta == 0), adv [B], mask [B, C] int32.
 * out3 = {loss, mean_kl, clip_ratio}; dlp [B, C] = d loss / d lp (may be NULL). One launch. */
int br_grpo_loss_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* adv,
                         const int32_t* mask, int B, int C, float beta, float eps_low, float eps_high,
                         float* out3, float* dlp, void* stream);
/* The same loss with truncated importance sampling against the rollout: rollout_lp [B, C] f32 = the sampler's log-probs
 * (br_sample_next*_logp).  Per token w = min(exp(o - rollout_lp), is_cap), o = old_lp (lp when NULL), a constant; the clipped
 * policy-gradient term is multiplied by w, the KL term is not.  is_cap > 0 (+inf: untruncated).  out3 as above;
 * is_stats[4] = masked token means of {w, [exp(o - rollout_lp) > is_cap], o - rollout_lp, exp(o - rollout_lp) - 1 - (o - rollout_lp)}.
 * One launch. */
int br_grpo_loss_is_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* rollout_lp, const float* adv,
                            const int32_t* mask, int B, int C, float beta, float eps_low, float eps_high, float is_cap, float* out3,
                            float* is_stats, float* dlp, void* stream);
/* The loss with high-entropy token selection (TRL's top_entropy_quantile, "Beyond the 80/20 Rule"): entropy [B, C] f32 per token
 * (br_lmhead_logprob_entropy_fwd), tau [1] f32 on the device (br_entropy_threshold).  A token's clipped policy-gradient term and its
 * gradient are kept only where mask && entropy >= *tau; the KL term, the per-row normalisation (sum of mask) and clip_ratio are
 * unchanged.  rollout_lp optional: non-NULL adds the truncated importance weight of br_grpo_loss_is_fwd_bwd (is_stats, is_cap as
 * there).  *tau = -inf reproduces br_grpo_loss_fwd_bwd / br_grpo_loss_is_fwd_bwd bit for bit.  ent_sum[1] = sum of mask * entropy.
 * One launch. */
int br_grpo_loss_ent_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* rollout_lp, const float* adv,
                             const int32_t* mask, const float* entropy, const float* tau, int B, int C, float beta, float eps_low,
                             float eps_high, float is_cap, float* out3, float* is_stats, float* ent_sum, float* dlp, void* stream);
/* tau[0] = torch.quantile(entropy[mask != 0], level) (linear interpolation) bit for bit, on the device (no host sync): entropy [n]
 * f32, mask [n] int32, level in [0, 1] (TRL: 1 - top_entropy_quantile).  Masked entries are not read as values.  No valid entry:
 * tau = +inf.  -0 is read as +0.  One launch. */
int br_entropy_threshold(const float* entropy, const int32_t* mask, int64_t n, float level, float* tau, void* stream);
/* completion_mask[b, t] = t <= first_eos(b) (grpo_trainer.py:605-609); ids int64 [B, C] -> mask int32 */
int br_eos_mask(const int64_t* completion_ids, int B, int C, int64_t eos_id, int32_t* mask, void* stream);

/* The GRPO objectives of later TRL releases (DESIGN.md §3).  Ratio: token level s = lp - o, or sequence level (GSPO) one
 * s_b = sum_t m (lp - o) / max(|o_b|, 1) per row; c1 = exp(s), c2 = clamp(c1, 1 - eps_low, 1 + eps_high), then c1 <- min(c1, delta)
 * (torch.clamp(max=delta)); per token l = -min(c1 A, c2 A) w k + beta k3, w the truncated importance weight of
 * br_grpo_loss_is_fwd_bwd (rollout_lp non-NULL), k the entropy keep-mask of br_grpo_loss_ent_fwd_bwd (entropy non-NULL).
 * Aggregation: norm_rows > 0 gives sum_b (sum_t m l / max(|o_b|, 1)) / norm_rows ("grpo"; norm_rows = the rows of the whole
 * local batch, so row chunks add up); norm_rows == 0 gives sum m l / *norm (norm [1] f32 on the device: bnpo, dr_grpo, dapo).
 * The outputs are sums, so row chunks add up without reweighting:
 *   out7 = {loss, sum_b of the row-mean k3 (rows with |o_b| > 0), sum m [c1 A < c2 A], sum m [c1 < 1 - eps_low && A < 0],
 *           sum m [c1 > 1 + eps_high && A > 0], sum m [either], sum m};
 *   is_sums[4] = the masked sums of br_grpo_loss_is_fwd_bwd's is_stats; ent_sum[1] = sum m * entropy.
 * With sequence_level = 0, delta = +inf and norm_rows = B, out7 / dlp carry br_grpo_loss*_fwd_bwd's bits.  One launch. */
typedef struct br_grpo_objective {
    int32_t sequence_level;       /* 0: per-token ratio; 1: one ratio per row */
    float delta;                  /* > 0; +inf: off */
    int32_t norm_rows;            /* > 0: "grpo" aggregation over that many rows; 0: divide by *norm */
    const float* norm;            /* [1] f32, device */
    const float* rollout_lp;      /* optional [B, C] f32 */
    float is_cap;                 /* > 0 when rollout_lp is given */
    float* is_sums;               /* [4], needed with rollout_lp */
    const float* entropy;         /* optional [B, C] f32 */
    const float* tau;             /* [1] f32, device, needed with entropy */
    float* ent_sum;               /* [1], needed with entropy */
} br_grpo_objective;
int br_grpo_objective_fwd_bwd(const float* lp, const float* old_lp, const float* ref_lp, const float* adv, const int32_t* mask, int B,
                              int C, float beta, float eps_low, float eps_high, const br_grpo_objective* opt, float* out7, float* dlp,
                              void* stream);
/* Advantages with TRL's scale_rewards: (r - group mean) / (std + 1e-4) with std the unbiased group std (GROUP: br_grpo_advantages'
 * bits), or the unbiased std of all rows (BATCH), or r - group mean (NONE).  std_used [rows] = the std of the row (the group std in
 * NONE mode), zero_std [rows] int32 = std_used <= 1e-8.  One launch (one CTA). */
#define BR_SCALE_REWARDS_GROUP 0
#define BR_SCALE_REWARDS_BATCH 1
#define BR_SCALE_REWARDS_NONE 2
int br_grpo_advantages_scaled(const float* rewards_per_func, int rows, int n_funcs, int G, int mode, float* advantages, float* std_used,
                              int32_t* zero_std, void* stream);
/* br_eos_mask with the rows that hold no EOS zeroed (mask_truncated_completions); lengths [B] int32 = each row's mask count before
 * that zeroing (min(first EOS + 1, C)).  A row with an EOS gets br_eos_mask's mask. */
int br_eos_mask_truncated(const int64_t* completion_ids, int B, int C, int64_t eos_id, int32_t* mask, int32_t* lengths, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense contractions on wgmma (replaces every nn.Linear / lm_head reached through
 * dna_llm.py:150-160,237-242; SURVEY.md §2.3 K1,K2,K5,K6,K7,K12)
 * ------------------------------------------------------------------------------------------- */
/* LoRA dropout (peft: y = base(x) + s * B(A(dropout(x)))) with a counter-based mask that is never stored: element (row, col) of the
 * input of projection j in decoder layer l, in pass c, is kept iff bits >= threshold, where
 *   w    = Philox4x32-10(counter = (col >> 3, row, (l << 3) | j, c), key = (seed mod 2^32, seed >> 32))
 *   bits = (w[(col & 7) >> 1] >> (16 * (col & 1))) & 0xFFFF
 * and kept elements are scaled by inv_keep.  row is the global token row (row_offset + local row), so chunked calls reproduce the
 * mask of the whole pass. */
typedef struct br_lora_dropout {
    uint64_t seed;
    uint32_t pass;           /* c: advanced once per dropout-applying pass */
    int32_t layer;           /* l */
    int32_t proj;            /* j of the first r-wide block (q 0, k 1, v 2, o 3, gate 4, up 5, down 6); block i is projection proj + i */
    int32_t r;               /* adapter rank: columns per projection (multiple of 16, <= 64) */
    int32_t threshold;       /* T = round(p * 65536), 1..65535 */
    float inv_keep;          /* 65536 / (65536 - T) */
    int64_t row_offset;      /* global token row of local row 0 */
} br_lora_dropout;

typedef struct br_gemm_epilogue {
    const void* bias;        /* [N] or NULL */
    int32_t bias_dtype;      /* BR_BF16 / BR_F32 */
    const void* residual;    /* bf16 [M, ldr] added after bias (indexed by OUTPUT row) or NULL */
    int64_t ldr;
    float alpha;             /* scales the accumulator first */
    int32_t act;             /* 0 none; 1: gated SiLU, columns in blocks of 16 = 8 gate | 8 up: out[:, 8b+i] = silu(acc[:, 16b+i]) * acc[:, 16b+8+i] */
    int32_t out_dtype;       /* BR_BF16 / BR_F32 */
    const int32_t* row_map;  /* optional [M]: output row of input row m (<0: dropped) -- projector scatter */
    void* aux_out;           /* act==1: optional bf16 [M, ld_aux] copy of the pre-activation accumulator */
    int64_t ld_aux;
    const void* A2;          /* optional second K segment accumulated into the same tile: */
    int64_t lda2;            /*   D += A2[M, K2] . B2[N, K2]^T   (LoRA delta, SURVEY.md K12) */
    const void* B2;
    int64_t ldb2;
    int32_t K2;
    const br_lora_dropout* lora_dropout;   /* optional (NULL: unmasked): the second segment is a LoRA up-path u . A; the product of
                                            each r-wide K block (projection proj + i) is multiplied by that projection's mask over
                                            [M, N] and by inv_keep before it joins the accumulator (dx of the dropped input) */
} br_gemm_epilogue;

/* D[M, N] = epilogue(A[M, K] . B[N, K]^T); A, B bf16 row-major (K contiguous); ld* in elements. */
int br_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd,
                 int M, int N, int K, const br_gemm_epilogue* epi, void* stream);

/* Fused lm_head + log-softmax + gather (replaces grpo_trainer.py:511-520 and HF loss_utils CE):
 * logp[m] = scale*H[m].W[target[m]] - logsumexp_v(scale*H[m].W[v]); logits never reach HBM.
 * target[m] < 0 => logp 0 (ignored row).  lse [M] is kept for the backward. */
int64_t br_lmhead_workspace_bytes(int M, int V);
int br_lmhead_logprob_fwd(const void* H, int64_t ldh, const void* W, int64_t ldw, const int32_t* target,
                          int M, int V, int K, float scale, float* logp, float* lse, void* workspace, void* stream);
/* br_lmhead_logprob_fwd plus the entropy of every row, target < 0 included:  entropy[m] = -sum_v p_v log p_v with
 * p = softmax_v(scale*H[m].W[v]).  logp and lse are bit-identical to br_lmhead_logprob_fwd's.  Workspace:
 * br_lmhead_entropy_workspace_bytes(M, V).  Two launches. */
int64_t br_lmhead_entropy_workspace_bytes(int M, int V);
int br_lmhead_logprob_entropy_fwd(const void* H, int64_t ldh, const void* W, int64_t ldw, const int32_t* target,
                                  int M, int V, int K, float scale, float* logp, float* lse, float* entropy, void* workspace,
                                  void* stream);
/* dlogits[m, v] = gscale[m] * (onehot(target[m])[v] - softmax(H[m].W)[v]) as bf16 [M, ldd] (recomputed tiles) */
int br_lmhead_dlogits(const void* H, int64_t ldh, const void* W, int64_t ldw, const int32_t* target,
                      const float* lse, const float* gscale, int M, int V, int K, float scale,
                      void* dlogits, int64_t ldd, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Row kernels (HBM-bound): norms, rotary, gathers  (replace HF Qwen3RMSNorm qwen3/modeling_qwen3.py:50-64,
 * torch LayerNorm in esm/modeling_esm.py:386-400,476-479,511, apply_rotary_pos_emb qwen3:120-150 / esm:45-55,
 * embed_tokens + masked scatter dna_llm.py:211-229)
 * ------------------------------------------------------------------------------------------- */
/* y = w * bf16(x * rsqrt(mean(x^2)+eps)); bf16 [M, d]; rstd [M] f32 optional (kept for the backward) */
int br_rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, float* rstd, int M, int d, float eps, void* stream);
int br_layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy, int M, int d, float eps, void* stream);
/* Pooled score head of a sequence-classification reward model (HF GenericForSequenceClassification): h bf16 [B*L, ldh] is the last
 * decoder layer's output BEFORE the final norm, input_ids int64 [B, L].  Per row: t = the rightmost column whose id != pad_id, over
 * all L columns (0 when every column is pad; pad_id = -1: none, t = L - 1); y = bf16(norm_w * bf16(h[t] * rsqrt(mean(h[t]^2) + eps)))
 * with an fp32 sum of squares; out[b * ldo + j] = float(bf16(sum_i y_i score_w[j, i])) with fp32 accumulation, j < n_labels.
 * index (NULL: not written) int32 [B] receives t.  d % 8 == 0, d <= 10240.  One launch, one CTA per row, fixed-order reductions:
 * the same bits on every launch. */
int br_seqcls_score(const void* h, int64_t ldh, const int64_t* input_ids, int B, int L, int64_t pad_id, const void* norm_w, float eps,
                    const void* score_w, int64_t ldw, int n_labels, int d, float* out, int64_t ldo, int32_t* index, void* stream);
/* In place on the fused QKV activation [M, ld]: heads 0..n_q-1 are queries, the next n_k are keys.
 * mode 0 (Qwen3): per-head RMSNorm with q_norm_w / k_norm_w [head_dim] (NULL = skip) then rotate-half RoPE;
 * mode 1 (ESM/NT-v2): queries scaled by q_scale, then RoPE.  positions [M] int32 (explicit: the reference uses
 * arange over the padded row in forward() and cumsum(mask)-1 in generate(), SURVEY.md §3.1/§3.2). */
int br_qk_rope(void* qkv, int64_t ld, int M, int n_q_heads, int n_k_heads, int head_dim, const void* q_norm_w,
               const void* k_norm_w, const int32_t* positions, float theta, float eps, float q_scale, int mode, void* stream);
/* same; out != NULL writes the roped q|k heads to out[M, >= (n_q+n_k)*head_dim] instead of in place (the pre-norm values stay in qkv for
 * the backward: no copy); rope_table (br_rope_table, [n_pos, head_dim/2] (cos, sin) pairs) replaces the per-element powf/sincosf (mode 0) */
int br_qk_rope_ex(void* qkv, int64_t ld, void* out, int64_t ldo, int M, int n_q_heads, int n_k_heads, int head_dim, const void* q_norm_w,
                  const void* k_norm_w, const int32_t* positions, float theta, float eps, float q_scale, int mode, const float* rope_table,
                  int rope_n_pos, void* stream);
/* out[m] = table[ids[m]] (zeros if keep && !keep[m], or id out of range); ids int64 */
int br_embed_gather(const int64_t* ids, const void* table, int64_t ldt, int64_t vocab, void* out, int64_t ldo, int M, int d,
                    const int32_t* keep, void* stream);
int br_scatter_rows(const void* src, int64_t lds, const int32_t* row_map, void* dst, int64_t ldd, int M, int d, void* stream);
/* out[m] = src[idx[m]] (idx < 0 -> zero row) */
int br_gather_rows(const void* src, int64_t lds, const int32_t* idx, void* dst, int64_t ldd, int M, int d, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Attention (replaces the SDPA call under Qwen3Attention / EsmSelfAttention; SURVEY.md K1, K5)
 * q/k/v/o bf16 token-major [B*L, ld] with head h at column h*head_dim; row b attends keys in
 * [kv_start[b], kv_end[b]) (NULL = whole row) and, if causal, j <= i.  lse [B, Hq, L] f32 optional.
 * ------------------------------------------------------------------------------------------- */
int br_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                float* lse, int B, int L, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* kv_start,
                const int32_t* kv_end, float scale, int causal, void* stream);
/* Shared-prefix layout (GRPO groups: G rows that repeat one prompt): U groups of G rows of L = Lp + Ls positions, Lp a multiple of 64.
 * The buffer holds [U * Lp prefix rows | R = U * G suffixes of Ls rows]: group u's positions 0 .. Lp-1 are rows u * Lp + t, row
 * r = u * G + g's position Lp + t is row U * Lp + r * Ls + t.  Causal, head_dim 128; kv_start [U] per group (the rows of a group share
 * their prompt), kv_end [R] per row, with kv_end >= Lp (every row's window reaches past the prefix).  The log-sum-exp is kept as two
 * segment buffers: lse_prefix [U, Hq, Lp] (unused when Lp = 0) and lse_suffix [R, Hq, Ls].  O and the log-sum-exp are bit-identical
 * to br_attn_fwd on the equivalent dense [R, L] rows. */
int br_attn_fwd_shared(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                       float* lse_prefix, float* lse_suffix, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads, int head_dim,
                       const int32_t* kv_start, const int32_t* kv_end, float scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Rollout / decode (replaces the HF generate() token loop, DynamicCache and logits warpers reached from
 * dna_llm.py:298-304; HF generation/utils.py:2760-2800, 1214-1223; SURVEY.md K8, K9)
 * KV cache per layer: K and V are [n_pages, Hkv, 64, head_dim] bf16; page_table int32 [R, max_pages];
 * cur_len int32 [R] = tokens already cached for the row (the position of the token being decoded).
 * ------------------------------------------------------------------------------------------- */
/* scratch of br_skinny_gemm for weights of up to max_N rows: zero-initialised once (its arrival counters self-reset) */
int64_t br_skinny_scratch_bytes(int max_N);
/* out[R, N] = X[R, K] . W[N, K]^T for R <= 32 (HBM-bound weight streaming). mode 0: bf16; 1: bf16(out) + residual;
 * 2: SwiGLU over (8 gate | 8 up) row blocks -> [R, N/2]; 3: fp32.
 * Folded RMSNorm for the decode step (norm weight pre-multiplied into W's columns by br_scale_columns), both optional (NULL):
 * sumsq_in [sumsq_in_n, 32]: partial sums of x^2 per row; out rows are scaled by rsqrt(sum_i sumsq_in[i, r] / K + eps);
 * sumsq_out [ceil(N/128)*4, 32]: partial sums of the bf16-rounded outputs squared (modes 0/1), one partial row per 32
 * features (so the consumer passes sumsq_in_n = ceil(N/128)*4).  No floating-point atomics: the rollout is reproducible. */
int br_skinny_gemm(const void* X, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, int R, int N, int K, int mode,
                   const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n, float* sumsq_out,
                   float eps, void* stream);
/* Weight-only FP8 (e4m3) for the rollout decode.  br_quantize_rows_e4m3: W [N, K] bf16 (row stride ldw, K % 16 == 0) ->
 * scale [N] fp32 = amax_k |W[n, k]| / 448 (1 for an all-zero row) and Q = e4m3fn(W[n, k] / scale[n]) (round to nearest even, never a
 * NaN code) in a private layout of br_fp8_weight_bytes(N, K) bytes (16-byte aligned) that only br_skinny_gemm_fp8 reads.
 * br_skinny_gemm_fp8: br_skinny_gemm with W = that buffer (ldw = K) and out[r, n] = scale[n] * (X . dequantized-codes^T)[r, n]
 * before the mode's epilogue (mode 2: gate and up features each with their own scale); same modes, statistics, scratch and
 * reproducibility. */
int64_t br_fp8_weight_bytes(int N, int K);
int br_quantize_rows_e4m3(const void* W, int64_t ldw, int N, int K, void* Q, float* scale, void* stream);
int br_skinny_gemm_fp8(const void* X, int64_t ldx, const void* W, int64_t ldw, const float* w_scale, void* out, int64_t ldo, int R, int N,
                       int K, int mode, const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n,
                       float* sumsq_out, float eps, void* stream);
int br_embed_gather_sumsq(const int64_t* ids, const void* table, int64_t ldt, int64_t vocab, void* out, int64_t ldo, int M, int d,
                          float* sumsq, void* stream);
/* W[n, k] *= scale[k] in place (bf16) */
int br_scale_columns(void* W, int64_t ld, int64_t N, int K, const void* scale, void* stream);
/* prefill: copy roped K / V of tokens [0, n_tok) of one prompt row (qkv points at its first real token) into pages[] */
int br_kv_write_pages(const void* qkv, int64_t ld, int n_tok, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* pages,
                      void* kcache, void* vcache, void* stream);
/* temperature -> top-k -> top-p -> inverse-CDF draw with uniforms[step*R + r] (or argmax when !do_sample); finished rows
 * emit pad_id; writes tokens[r, step] (int64 [R, max_steps]) when step < max_steps and next_ids[r]; eos_id < 0 disables EOS.
 * top_k is clamped to V; every value equal to the k-th is kept (HF's rule) up to 1024 kept values, past that the ties with the
 * lowest token ids. */
int br_sample_next(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                   const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                   int64_t* tokens, int64_t* next_ids, void* stream);
/* Same semantics in two stages for large vocabularies: stage 1 (V/4096 CTAs per row) reduces each row to <= 64 candidates
 * per 4096-logit chunk, stage 2 samples from the candidates (top_k <= 32), or from the logits row when a chunk held more ties
 * of its k-th value than that.  The workspace holds the candidates and one overflow flag per chunk. */
int64_t br_sample_workspace_bytes(int R, int V);
int br_sample_next_2stage(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                          const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id,
                          int32_t* finished, int64_t* tokens, int64_t* next_ids, void* workspace, void* stream);
/* The two samplers above that also write the behaviour log-prob logp[r, step] (f32, laid out like tokens) = z[y] - logsumexp(z)
 * over the raw logits row z (T = 1, full vocabulary, no top-k / top-p) at the chosen token y; finished rows write 0.  The
 * two-stage one needs br_sample_logp_workspace_bytes(R, V): br_sample_workspace_bytes(R, V) followed by R * ceil(V / 4096)
 * (max, sum exp) float pairs that stage 1 writes per chunk.  Tokens equal those of the calls without logp. */
int64_t br_sample_logp_workspace_bytes(int R, int V);
int br_sample_next_logp(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                        const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                        int64_t* tokens, int64_t* next_ids, float* logp, void* stream);
int br_sample_next_2stage_logp(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                               const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id,
                               int32_t* finished, int64_t* tokens, int64_t* next_ids, float* logp, void* workspace, void* stream);
/* Logits processors of the processed samplers (HF generation/logits_process.py), applied in HF's order on the fp32 logits row z:
 *   repetition penalty theta: z_j = z_j < 0 ? z_j * theta : z_j / theta (fp32, IEEE division) for each distinct token j whose bit is set
 *     in presence[r] (bit j % 32 of word j / 32 of row r; the bitmap is [R, ceil(V / 32)] uint32, contiguous);
 *   min_new_tokens m: z[eos_id] = -inf while *step < m (step NULL: 0; nothing when eos_id < 0);
 *   then temperature -> top-k -> top-p as above, then min-p: drop every kept token with exp((z_j - z_max) / T) < min_p (the maximum
 *     always stays).  Greedy (!do_sample) takes the argmax of the penalised, EOS-masked row; T, top-k, top-p and min_p do nothing there.
 * After the draw each row sets the bit of the token it emits (pad for a finished row).  The caller zeroes presence before a sequence's
 * first draw; presence may be NULL only when repetition_penalty == 1 (then nothing is penalised or recorded).  Refused: theta <= 0,
 * min_p outside [0, 1], min_new_tokens < 0.  logp (NULL: none) is the behaviour log-prob of the *_logp entry points: the RAW logits
 * (T = 1, full vocabulary, no processor) at the chosen token; the two-stage one then needs br_sample_logp_workspace_bytes.  With
 * theta = 1, min_p = 0 and m = 0 the tokens and logp equal those of the entry points above. */
typedef struct br_sample_proc {
    float repetition_penalty;    /* theta > 0; 1: off */
    float min_p;                 /* [0, 1]; 0: off */
    int32_t min_new_tokens;      /* m >= 0; 0: off */
    uint32_t* presence;          /* [R, ceil(V / 32)] emitted-token bitmap, read before and updated after the draw */
} br_sample_proc;
int br_sample_next_proc(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                        const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id, int32_t* finished,
                        int64_t* tokens, int64_t* next_ids, float* logp, const br_sample_proc* proc, void* stream);
int br_sample_next_2stage_proc(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, int do_sample,
                               const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id,
                               int32_t* finished, int64_t* tokens, int64_t* next_ids, float* logp, const br_sample_proc* proc,
                               void* workspace, void* stream);
/* Full-vocabulary sampler: the draw above without the 1024-value cap, for any top_k >= 0 (0: top-k off).  z' is z after the
 * processors of proc (NULL: none; min_p, repetition_penalty and min_new_tokens as above).  top_k >= 1 is clamped to V and keeps every
 * value >= the k-th, ties included, with no cap; top-p orders the kept tokens by value desc, id asc, drops from the end while the
 * cumulative probability at T is <= 1 - p (always keeping the first; among equal values the higher ids go first); min-p then drops
 * exp((z'_j - z'_max) / T) < min_p; the draw is the inverse CDF over the kept tokens in ascending id.  Weights are
 * exp((z' - max) / T), computed in fp64 and held as 64-bit fixed point (2^-40): the cuts and the draw are exact integer arithmetic on them.  logp (NULL: none)
 * as in the *_logp entry points, bit-equal to br_sample_next_2stage_logp's for the same token.  A row with no finite z' draws pad_id.
 * Refused: T <= 0, top_p <= 0, top_k < 0, no uniforms, V >= 2^23, and what the processed entry points refuse.  workspace:
 * br_sample_full_workspace_bytes(R, V), no initialisation needed (the first kernel resets it).  Up to 8 kernels, chained with PDL; the
 * sequence depends on (top_k, top_p) only, so a captured graph replays it. */
int64_t br_sample_full_workspace_bytes(int R, int V);
int br_sample_next_full(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p,
                        const float* uniforms, const int32_t* step, int max_steps, int64_t eos_id, int64_t pad_id,
                        int32_t* finished, int64_t* tokens, int64_t* next_ids, float* logp, const br_sample_proc* proc,
                        void* workspace, void* stream);
int br_decode_advance(int32_t* step, int32_t* cur_len, int R, void* stream);

/* Decode attention, one launch per layer per step: per-head q/k RMSNorm + RoPE at cur_len[r], K/V append to the row's page,
 * paged attention and split merge.  qkv_raw is the un-normalised fused projection of the new tokens.  Rows are R/G groups whose
 * first n_shared_pages table entries are identical (prefix sharing: the shared pass reads each prompt K/V tile once per group);
 * G * n_q_heads/n_kv_heads <= 32.  splits_shared + splits_private <= 32 partial slots per head.  rope_table (br_rope_table,
 * covering every position of the rollout) is required.  workspace: br_decode_fused_workspace_bytes, zero-initialised once
 * (arrival counters are self-resetting). */
int64_t br_decode_fused_workspace_bytes(int R, int n_q_heads, int n_kv_heads, int head_dim, int n_slots);
int br_decode_attn_fused(const void* qkv_raw, int64_t ld, const void* q_norm_w, const void* k_norm_w, void* kcache, void* vcache,
                         const int32_t* page_table, int max_pages, const int32_t* cur_len, int R, int G, int n_q_heads,
                         int n_kv_heads, int head_dim, int n_shared_pages, int splits_shared, int splits_private, float scale,
                         float theta, float eps, const float* rope_table, int rope_n_pos, void* workspace, void* out, int64_t ldo,
                         void* stream);
/* rope_table [n_pos, head_dim/2, 2] f32 = (cos, sin) rounded to bf16 precision (HF builds its tables in the model dtype);
 * input of br_decode_attn_fused: removes powf/sincosf from the decode loop. */
int br_rope_table(float* out, int n_pos, int head_dim, float theta, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Backward (autograd counterparts; frozen base weights + LoRA adapters, reason.py:362-394; SURVEY.md K12)
 * ------------------------------------------------------------------------------------------- */
int64_t br_attn_bwd_workspace_bytes(int B, int L, int n_q_heads, int head_dim);
/* dq/dk/dv (bf16, strided -- typically the three column blocks of one fused dqkv buffer) from dout; causal, head_dim 128 */
int br_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                const void* dout, int64_t lddo, const float* lse, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv,
                int64_t lddv, int B, int L, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* kv_start,
                const int32_t* kv_end, float scale, void* workspace, void* stream);
/* Backward of br_attn_fwd_shared (same layout and windows).  dQ of every query and dK / dV of the suffix keys are bit-identical to
 * br_attn_bwd on the dense rows; the prefix dK / dV sum the group's prefix queries, then the queries of rows g = 0 .. G-1 in that order
 * (bit-identical to the dense result when G = 1).  No atomics: bit-reproducible.  workspace: br_attn_bwd_shared_workspace_bytes. */
int64_t br_attn_bwd_shared_workspace_bytes(int U, int G, int Lp, int Ls, int n_q_heads, int head_dim);
int br_attn_bwd_shared(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                       const void* dout, int64_t lddo, const float* lse_prefix, const float* lse_suffix, void* dq, int64_t lddq, void* dk,
                       int64_t lddk, void* dv, int64_t lddv, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads, int head_dim,
                       const int32_t* kv_start, const int32_t* kv_end, float scale, void* workspace, void* stream);
/* dx = d(RMSNorm)/dx . dy (+ dres): x, dy, dres, dx bf16 [M, d]; rstd from the forward */
int br_rmsnorm_bwd(const void* x, int64_t ldx, const void* w, const float* rstd, const void* dy, int64_t lddy, const void* dres,
                   int64_t lddr, void* dx, int64_t lddx, int M, int d, void* stream);
/* gu, dgu [M, 2F] in the blocked (8 gate | 8 up) layout; dact [M, F] */
int br_swiglu_bwd(const void* gu, int64_t ldgu, const void* dact, int64_t ldda, void* dgu, int64_t lddgu, int M, int F, void* stream);
/* in place on the q and k head columns of dqkv: inverse RoPE then per-head RMSNorm backward (qk_pre = pre-norm q|k) */
int br_qk_rope_bwd(void* dqkv, int64_t ldd, const void* qk_pre, int64_t ldp, int M, int n_q_heads, int n_k_heads, int head_dim,
                   const void* q_norm_w, const void* k_norm_w, const int32_t* positions, float theta, float eps, void* stream);
/* LoRA weight gradients on wgmma (deterministic):  product[P, N] = big[M, P]^T . small[M, N] over the M tokens (both token-major,
 * bf16, read as MN-major tensor-core operands), then  dst (+)= the blocks the segments name.
 *   mode 0: segment i adds product rows [row_lo, row_hi), columns [col_lo, col_lo + n_cols) into dst[(row - row_lo) * ld + col - col_lo]
 *           (dB of one adapter, or the q / k / v blocks of the fused qkv product);
 *   mode 1: one segment, transposed: dst[n * ld + p] += product[p, n]  (dA = u^T x written as [r, in]);
 *   mode 2: gate/up-blocked rows (16 = 8 gate | 8 up): segment 0 takes the gate rows, segment 1 the up rows -> dst row (p / 16) * 8 + p % 8.
 * workspace: br_lora_grad_workspace_bytes(), zero-initialised once.  Replaces torch autograd through peft's LoRA Linear (reason.py:362-394). */
typedef struct br_lora_grad_seg { float* dst; int64_t ld; int32_t row_lo, row_hi, col_lo, n_cols; } br_lora_grad_seg;
int64_t br_lora_grad_workspace_bytes(void);
int br_lora_grad_tn(const void* big, int64_t ldb, const void* small, int64_t lds, int M, int P, int N, int mode,
                    const br_lora_grad_seg* segs, int n_seg, void* workspace, void* stream);
/* Same product with the dropout mask of projection d->proj applied to `big` (features = mask columns, tokens = mask rows) and the
 * result scaled by d->inv_keep: dA = inv_keep * u^T (x . m) for one adapter (mode 1). */
int br_lora_grad_tn_dropout(const void* big, int64_t ldb, const void* small, int64_t lds, int M, int P, int N, int mode,
                            const br_lora_grad_seg* segs, int n_seg, const br_lora_dropout* d, void* workspace, void* stream);
/* LoRA down-projection with dropout (forward): t[M, n_proj * r] = scale * inv_keep * ((x . m_j) . A_j^T) for the n_proj stacked
 * adapters A [n_proj * r, K] of one fused linear (j = d->proj + block), bf16 out; x is read once for all of them. */
int br_lora_down_dropout(const void* x, int64_t ldx, const void* A, int64_t lda, void* t, int64_t ldt, int M, int K, int n_proj,
                         float scale, const br_lora_dropout* d, void* stream);
/* keep[m, k] = 1 if element (row_offset + m, k) of projection d->proj's input is kept, else 0 (uint8 [M, ldo]; tests / inspection) */
int br_lora_dropout_mask(const br_lora_dropout* d, int M, int K, uint8_t* keep, int64_t ldo, void* stream);
int br_transpose_bf16(const void* in, int64_t ldi, void* out, int64_t ldo, int M, int N, void* stream);
int br_colsum_accumulate(const void* in, int64_t ldi, float* out, int M, int N, void* stream);

#ifdef __cplusplus
}
#endif
#endif
