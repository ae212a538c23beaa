// LoRA dropout masks in registers (the rule is spelled out next to br_lora_dropout in include/bioreason_b200.h).
// One Philox4x32-10 call gives the 16-bit draws of 8 consecutive columns of one row, so the four lanes of a quad in the wgmma fragment
// layout (same row, column pairs 2q, 2q + 1 of every 8-column group) cover four (row, 8-column) groups with one call each and trade
// words through quad_words(): no call is made twice and nothing is stored.
#pragma once
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"

namespace br {

struct DropParams {
    uint32_t k0, k1, pass;
    int layer, proj, r, T;
    float inv_keep;
    long long row0;
};

static inline DropParams drop_params(const br_lora_dropout& d) {
    DropParams p;
    p.k0 = (uint32_t)(d.seed & 0xFFFFFFFFull); p.k1 = (uint32_t)(d.seed >> 32); p.pass = d.pass;
    p.layer = d.layer; p.proj = d.proj; p.r = d.r; p.T = d.threshold; p.inv_keep = d.inv_keep; p.row0 = d.row_offset;
    return p;
}

static inline int check_drop(const br_lora_dropout* d, const char* who) {
    BR_CHECK_ARG(d != nullptr, "%s: dropout descriptor is NULL", who);
    BR_CHECK_ARG(d->threshold >= 1 && d->threshold <= 65535, "%s: threshold %d outside [1, 65535]", who, d->threshold);
    BR_CHECK_ARG(d->layer >= 0 && d->proj >= 0 && d->proj < 8 && d->row_offset >= 0, "%s: bad layer / projection / row offset", who);
    return BR_OK;
}

#ifdef __CUDACC__
// 128 random bits of the group (row, columns 8 cg .. 8 cg + 7) of projection j
__device__ __forceinline__ uint4 drop_group(const DropParams& d, long long row, int cg, int j) {
    return philox4x32_10(make_uint4((uint32_t)cg, (uint32_t)row, ((uint32_t)d.layer << 3) | (uint32_t)j, d.pass), d.k0, d.k1);
}

__device__ __forceinline__ uint32_t sel4(uint4 w, int i) { return i == 0 ? w.x : i == 1 ? w.y : i == 2 ? w.z : w.w; }

// Lane q of a quad passes the words of ITS group (group q of the quad's four); returns in out[i] word q of group i.
__device__ __forceinline__ void quad_words(uint4 w, uint32_t (&out)[4]) {
    const int lane = threadIdx.x & 31, q = lane & 3;
    uint32_t got[4];
#pragma unroll
    for (int t = 0; t < 4; ++t)                     // step t: lane q reads group (q + t) & 3, whose owner sends word (owner - t) & 3 = q
        got[t] = __shfl_sync(0xffffffffu, sel4(w, (q - t) & 3), (lane & ~3) | ((q + t) & 3));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = (i - q) & 3;
        out[i] = t == 0 ? got[0] : t == 1 ? got[1] : t == 2 ? got[2] : got[3];
    }
}

// bf16-pair mask of one 32-bit word: low half = even column, high half = odd column; all-ones where the element is kept
__device__ __forceinline__ uint32_t keep_bits(uint32_t w, int T) {
    return ((w & 0xFFFFu) >= (uint32_t)T ? 0x0000FFFFu : 0u) | ((w >> 16) >= (uint32_t)T ? 0xFFFF0000u : 0u);
}
__device__ __forceinline__ bool keep_lo(uint32_t w, int T) { return (w & 0xFFFFu) >= (uint32_t)T; }
__device__ __forceinline__ bool keep_hi(uint32_t w, int T) { return (w >> 16) >= (uint32_t)T; }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
#endif

}  // namespace br
