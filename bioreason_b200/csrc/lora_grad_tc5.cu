// LoRA weight gradients on wgmma (sm_90a):  out (+)= big[M, P]^T . small[M, N]   (contraction over the M tokens; fp32 out, N <= 128).
//
// Autograd of the adapters the reference trains with peft (reason.py:362-394): dB = dy^T t and dA = u^T x (SURVEY.md §2.3 K12).
// Both operands are read exactly as the forward/backward left them -- token-major [M, features] -- as MN-MAJOR wgmma operands
// (the TMA box [64 tokens x 64 features] is one swizzle atom column; no transposed copies).  One launch covers a whole fused linear:
// the full [P, N] product of e.g. dqkv^T (6144 features) with t_qkv (3r columns) is formed in registers and the epilogue writes only the
// block each adapter owns (q rows x its r columns, ...), so 14 launches per decoder layer become 8.
// Split-K over the token dimension fills the SMs for narrow outputs; partial tiles are exchanged through a workspace and summed
// by the split-0 CTA in ascending split order (release/acquire counter, no floating-point atomics): gradients are bit-reproducible.
// With LoRA dropout (MASK, dA = inv_keep * u^T (x . m)): the MN-major `big` tile is loaded into register fragments (ldmatrix.trans),
// ANDed with the counter-based mask and fed to the register-A wgmma; each lane draws one (token, 8-feature) group per k16 step and the
// warp trades the 16-bit draws through 512 bytes of shared memory.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "lora_dropout.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128, BKT = 64, NTHREADS = 160, NSTAGE = 4;   // warps 0..3: wgmma + epilogue, warp 4: TMA
constexpr int A_BYTES = 2 * 64 * 128;          // two [64 tokens x 64 features] blocks
constexpr int B_BLK = 64 * 128;

struct Seg { float* dst; long long ld; int row_lo, row_hi, col_lo, n_cols; };   // rows [row_lo,row_hi) of the product, columns [col_lo, col_lo+n_cols)

struct TnParams {
    int M, P, N, Npad, NBB;                    // NBB = 64-column blocks of `small`
    int tiles, splits, kb_total;
    int mode;                                  // 0: segments (row-major dst[(p - row_lo) * ld + n]); 1: transposed dst[n * ld + p];
                                               // 2: gate/up interleave: product row p = block of 16 = 8 gate | 8 up -> dst rows (p/16)*8 + p%8
    Seg seg[3]; int n_seg;
    float* ws; int* counters;
    br::DropParams drop;                       // MASK only
};

// Masked A fragment (features 16 w.. of one 64-feature block x tokens t0 + 0..15): a[i] = feature + 8 (i & 1), tokens + 8 (i >> 1) + 2q, +1
__device__ __forceinline__ void masked_big_frag(uint32_t (&a)[4], uint32_t blk, int kk, long long tok0, int feat0, const br::DropParams& d,
                                                uint4* xbuf) {
    const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3, mi = lane >> 3;
    const int tok = kk * 16 + (lane & 7) + ((mi >> 1) << 3);
    const int chunk = 2 * warp + (mi & 1);
    br::ldsm_x4_t(a, blk + tok * 128 + ((chunk ^ (lane & 7)) << 4));
    // lane L draws group (token tok0 + (L & 15), features 8 ((feat0 >> 3) + (L >> 4)) ..)
    xbuf[lane] = br::drop_group(d, tok0 + (lane & 15), (feat0 >> 3) + (lane >> 4), d.proj);
    __syncwarp();
    const uint16_t* b16 = reinterpret_cast<const uint16_t*>(xbuf);
    const int fe = (lane >> 2) & 7, q = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int g = 8 * (i >> 1) + 2 * q + 16 * (i & 1);
        a[i] &= br::keep_bits((uint32_t)b16[g * 8 + fe] | ((uint32_t)b16[(g + 1) * 8 + fe] << 16), d.T);   // tokens 2q | 2q + 1
    }
    __syncwarp();
}

template <int NPAD, bool MASK>
__global__ void __launch_bounds__(NTHREADS, 1)
tn_gemm_tc5_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TnParams p) {
    constexpr int NBB = NPAD / 64;
    constexpr int STAGE = A_BYTES + NBB * B_BLK;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE);
    uint64_t* empty_bar = full_bar + NSTAGE;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x / p.splits, split = blockIdx.x % p.splits;
    const int kb_per = (p.kb_total + p.splits - 1) / p.splits;
    const int kb_lo = split * kb_per, kb_hi = min(p.kb_total, kb_lo + kb_per);
    const int n_kb = max(0, kb_hi - kb_lo);

    if (threadIdx.x == 0) {
        br::tma_prefetch_desc(&tmA); br::tma_prefetch_desc(&tmB);
        for (int s = 0; s < NSTAGE; ++s) { br::mbar_init(&full_bar[s], 1); br::mbar_init(&empty_bar[s], 1); }
        br::mbar_fence_init();
    }
    __syncthreads();

    if (warp == 4) {
        if (lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int kb = kb_lo; kb < kb_hi; ++kb) {
                br::mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* sa = smem + s * STAGE;
                br::mbar_expect_tx(&full_bar[s], STAGE);
                br::tma_load_2d(sa, &tmA, &full_bar[s], tile * BM, kb * BKT);
                br::tma_load_2d(sa + 64 * 128, &tmA, &full_bar[s], tile * BM + 64, kb * BKT);
#pragma unroll
                for (int nb = 0; nb < NBB; ++nb) br::tma_load_2d(sa + A_BYTES + nb * B_BLK, &tmB, &full_bar[s], nb * 64, kb * BKT);
                if (++s == NSTAGE) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    // ---- one consumer warpgroup: two m64 products (features 0..63 and 64..127 of the tile), both operands MN-major
    const int et = threadIdx.x;                                          // 0..127
    const int row = et;                                                  // product row of this thread in the epilogue
    const int prow = tile * BM + row;                                    // row of the product = feature index of `big`
    float v[NPAD];
    if (n_kb > 0) {
        float acc0[NPAD / 2], acc1[NPAD / 2];
#pragma unroll
        for (int i = 0; i < NPAD / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
        int s = 0; uint32_t ph = 0;
        for (int i = 0; i < n_kb; ++i) {
            br::mbar_wait(&full_bar[s], ph);
            const uint32_t sa = br::smem_u32(smem + s * STAGE);
            br::wg_fence();
#pragma unroll
            for (int kk = 0; kk < BKT / 16; ++kk) {
                // 16 tokens = 2 groups of 8 rows (SBO 1024 B); 64-wide feature / column blocks are 8192 B apart (LBO)
                const uint64_t bd = br::wg_desc_mn(sa + A_BYTES + kk * 2048, B_BLK, 1024);
                if constexpr (MASK) {
                    uint4* xbuf = reinterpret_cast<uint4*>(smem + NSTAGE * STAGE + 256) + 32 * warp;
                    const long long tok0 = p.drop.row0 + (long long)(kb_lo + i) * BKT + kk * 16;
                    uint32_t a0[4], a1[4];
                    masked_big_frag(a0, sa, kk, tok0, tile * BM + 16 * warp, p.drop, xbuf);
                    masked_big_frag(a1, sa + 64 * 128, kk, tok0, tile * BM + 64 + 16 * warp, p.drop, xbuf);
                    br::wg_fence();
                    br::wgmma_rs<NPAD, 1>(acc0, a0, bd, 1);
                    br::wgmma_rs<NPAD, 1>(acc1, a1, bd, 1);
                } else {
                    br::wgmma_ss<NPAD, 1, 1>(acc0, br::wg_desc_mn(sa + kk * 2048, 64 * 128, 1024), bd, 1);
                    br::wgmma_ss<NPAD, 1, 1>(acc1, br::wg_desc_mn(sa + 64 * 128 + kk * 2048, 64 * 128, 1024), bd, 1);
                }
            }
            br::wg_commit();
            br::wg_wait<0>();
            if (et == 0) br::mbar_arrive(&empty_bar[s]);
            if (++s == NSTAGE) { s = 0; ph ^= 1; }
        }
        br::wg_fence_operand(acc0);
        br::wg_fence_operand(acc1);
        if constexpr (MASK) {
#pragma unroll
            for (int c = 0; c < NPAD / 2; ++c) { acc0[c] *= p.drop.inv_keep; acc1[c] *= p.drop.inv_keep; }
        }
        // every stage has been consumed and no load is in flight: the ring becomes the transpose buffer (one product row per thread)
        float* s_t = reinterpret_cast<float*>(smem);
        const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < NPAD / 8; ++i)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    s_t[(fr + 8 * hh) * (NPAD + 1) + 8 * i + fc + e] = acc0[4 * i + 2 * hh + e];
                    s_t[(64 + fr + 8 * hh) * (NPAD + 1) + 8 * i + fc + e] = acc1[4 * i + 2 * hh + e];
                }
        asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
        for (int c = 0; c < NPAD; ++c) v[c] = s_t[row * (NPAD + 1) + c];
    } else {
#pragma unroll
        for (int c = 0; c < NPAD; ++c) v[c] = 0.f;
    }
    {
        if (split != 0) {
            float* mine = p.ws + ((long long)blockIdx.x * NPAD) * BM + row;
#pragma unroll
            for (int c = 0; c < NPAD; ++c) __stcg(mine + c * BM, v[c]);
            __syncwarp();
            if (lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p.counters + tile) : "memory");
        } else {
            if (p.splits > 1) {
                if (et == 0) {
                    const unsigned want = 4u * (unsigned)(p.splits - 1);
                    unsigned seen;
                    do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(p.counters + tile) : "memory"); } while (seen < want);
                    p.counters[tile] = 0;
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");
                for (int s2 = 1; s2 < p.splits; ++s2) {                       // ascending split order: deterministic
                    const float* src = p.ws + ((long long)(tile * p.splits + s2) * NPAD) * BM + row;
#pragma unroll
                    for (int c = 0; c < NPAD; ++c) v[c] += __ldcg(src + c * BM);
                }
            }
            if (prow < p.P) {
                if (p.mode == 1) {
                    float* d = p.seg[0].dst + prow;
#pragma unroll
                    for (int c = 0; c < NPAD; ++c)
                        if (c < p.N) d[(long long)c * p.seg[0].ld] += v[c];
                } else {
#pragma unroll
                    for (int sgi = 0; sgi < 3; ++sgi) {
                        if (sgi >= p.n_seg) break;
                        const Seg& sg = p.seg[sgi];
                        int drow;
                        if (p.mode == 2) {                                    // gate/up interleave: seg 0 = gate rows, seg 1 = up rows
                            if (((prow >> 3) & 1) != sgi) continue;
                            drow = (prow >> 4) * 8 + (prow & 7);
                        } else {
                            if (prow < sg.row_lo || prow >= sg.row_hi) continue;
                            drow = prow - sg.row_lo;
                        }
                        float* d = sg.dst + (long long)drow * sg.ld;
#pragma unroll
                        for (int c = 0; c < NPAD; ++c)
                            if (c >= sg.col_lo && c < sg.col_lo + sg.n_cols) d[c - sg.col_lo] += v[c];
                    }
                }
            }
        }
    }
}

template <int NPAD, bool MASK = false>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const TnParams& p, cudaStream_t st) {
    constexpr int NBB = NPAD / 64;
    constexpr int SMEM = NSTAGE * (A_BYTES + NBB * B_BLK) + 256 + (MASK ? 4 * 32 * 16 : 0) + 1024;   // + the masked draw exchange
    static_assert(NSTAGE * (A_BYTES + NBB * B_BLK) >= BM * (NPAD + 1) * 4, "transpose buffer");
    auto kern = tn_gemm_tc5_kernel<NPAD, MASK>;
    static bool done = false;
    if (!done) { BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM)); done = true; }
    kern<<<p.tiles * p.splits, NTHREADS, SMEM, st>>>(ta, tb, p);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // namespace

extern "C" {

int64_t br_lora_grad_workspace_bytes(void) {
    // partial tiles [n_sms][128 cols][128 rows] fp32 + one counter per 128-feature tile (zero-initialised once; self-resetting)
    return (int64_t)br_num_sms() * 128 * BM * sizeof(float) + 4096 * sizeof(int);
}

static int lora_grad_tn(const void* big, int64_t ldb, const void* small, int64_t lds, int M, int P, int N, int mode,
                        const br_lora_grad_seg* segs, int n_seg, const br_lora_dropout* d, void* workspace, void* stream) {
    BR_CHECK_ARG(M > 0 && P > 0 && N >= 8 && N <= 128 && N % 8 == 0, "lora_grad_tn: M=%d P=%d N=%d (N %% 8, <= 128)", M, P, N);
    BR_CHECK_ARG(P % 8 == 0 && ldb % 8 == 0 && lds % 8 == 0 && ((uintptr_t)big % 16 == 0) && ((uintptr_t)small % 16 == 0), "lora_grad_tn: alignment");
    BR_CHECK_ARG(mode >= 0 && mode <= 2 && n_seg >= 1 && n_seg <= 3 && segs && workspace, "lora_grad_tn: bad mode / segments");
    BR_CHECK_ARG((P + BM - 1) / BM <= 4096, "lora_grad_tn: P too large");
    TnParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.P = P; p.N = N; p.mode = mode; p.n_seg = n_seg;
    for (int i = 0; i < n_seg; ++i) {
        p.seg[i].dst = segs[i].dst; p.seg[i].ld = segs[i].ld; p.seg[i].row_lo = segs[i].row_lo; p.seg[i].row_hi = segs[i].row_hi;
        p.seg[i].col_lo = segs[i].col_lo; p.seg[i].n_cols = segs[i].n_cols;
        BR_CHECK_ARG(segs[i].dst && segs[i].col_lo >= 0 && segs[i].col_lo + segs[i].n_cols <= N, "lora_grad_tn: segment %d columns outside [0, N)", i);
    }
    p.Npad = N <= 64 ? 64 : 128;                                  // MN-major wgmma operands come in 64-column swizzle atoms
    p.tiles = (P + BM - 1) / BM;
    p.kb_total = (M + BKT - 1) / BKT;
    int splits = br_num_sms() / p.tiles;                        // every CTA must be co-resident (the reducer spins on its peers)
    if (splits < 1) splits = 1;
    if (splits > 16) splits = 16;
    if (splits > p.kb_total) splits = p.kb_total;
    if (p.tiles > br_num_sms()) splits = 1;                     // more tiles than SMs: whole-K tiles, no exchange
    p.splits = splits;
    p.ws = (float*)workspace;
    p.counters = (int*)(p.ws + (int64_t)br_num_sms() * 128 * BM);
    CUtensorMap ta, tb;
    int rc;
    // token-major matrices, box = [64 tokens x 64 features]: tokens beyond M and features beyond the row are zero-filled by TMA
    if ((rc = br_make_tmap_2d_bf16(&ta, big, (uint64_t)M, (uint64_t)P, (uint64_t)ldb, BKT))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tb, small, (uint64_t)M, (uint64_t)N, (uint64_t)lds, BKT))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (d) {
        p.drop = br::drop_params(*d);
        return p.Npad == 64 ? launch<64, true>(ta, tb, p, st) : launch<128, true>(ta, tb, p, st);
    }
    return p.Npad == 64 ? launch<64>(ta, tb, p, st) : launch<128>(ta, tb, p, st);
}

int br_lora_grad_tn(const void* big, int64_t ldb, const void* small, int64_t lds, int M, int P, int N, int mode,
                    const br_lora_grad_seg* segs, int n_seg, void* workspace, void* stream) {
    return lora_grad_tn(big, ldb, small, lds, M, P, N, mode, segs, n_seg, nullptr, workspace, stream);
}

int br_lora_grad_tn_dropout(const void* big, int64_t ldb, const void* small, int64_t lds, int M, int P, int N, int mode,
                            const br_lora_grad_seg* segs, int n_seg, const br_lora_dropout* d, void* workspace, void* stream) {
    int rc;
    if ((rc = br::check_drop(d, "lora_grad_tn_dropout"))) return rc;
    return lora_grad_tn(big, ldb, small, lds, M, P, N, mode, segs, n_seg, d, workspace, stream);
}

}  // extern "C"
