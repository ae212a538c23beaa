// Shared device/host helpers for libbioreason_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#define BR_OK 0
#define BR_ERR_INVALID (-1)
#define BR_ERR_CUDA (-2)
#define BR_ERR_UNSUPPORTED (-3)

void br_set_error(const char* fmt, ...);

#define BR_CHECK_ARG(cond, ...)                     \
    do {                                            \
        if (!(cond)) {                              \
            br_set_error(__VA_ARGS__);              \
            return BR_ERR_INVALID;                  \
        }                                           \
    } while (0)

#define BR_CHECK_CUDA(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            br_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return BR_ERR_CUDA;                                                          \
        }                                                                                \
    } while (0)

// launch errors are collected without synchronising (SURVEY.md §8b error contract)
#define BR_CHECK_LAUNCH() BR_CHECK_CUDA(cudaGetLastError())

static inline int br_num_sms() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

#ifdef __CUDACC__
namespace br {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// ---------------- mbarrier ----------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---------------- TMA ----------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// same with an L2 eviction-priority hint (policy from make_policy_evict_first)
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}
// contiguous bulk copy global -> shared (bytes and both addresses 16-byte aligned), same completion and hint as above
__device__ __forceinline__ void bulk_load_hint(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(smem_dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t make_policy_evict_first() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}

// generic-proxy shared-memory writes -> visible to the async proxy (wgmma / TMA reading shared memory)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------- programmatic dependent launch (PDL) ----------------
// launch_dependents: lets the NEXT kernel in the stream start its prologue (barrier init, weight prefetch)
// while this one is still running; grid_dep_wait: blocks until the PREVIOUS kernel has completed and flushed memory.
// Everything that reads or writes data shared with earlier kernels must come after grid_dep_wait().
__device__ __forceinline__ void launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------- misc ----------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    bf162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t v) {
    bf162 t = *reinterpret_cast<bf162*>(&v);
    return __bfloat1622float2(t);
}

// ---------------- counter-based random numbers ----------------
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): ten rounds of two 32x32->64-bit
// multiplies with a Weyl-sequence key schedule.  Stateless: the same (counter, key) gives the same 128 bits on any thread.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        if (i) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

}  // namespace br
#endif

#ifdef __CUDACC__
// Launch with the programmatic-stream-serialization attribute (the kernel must call br::grid_dep_wait()).
template <typename... KArgs, typename... Args>
static inline cudaError_t br_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    static const bool no_pdl = getenv("BR_NO_PDL") != nullptr;          // debugging switch: plain stream-ordered launches
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = no_pdl ? 0 : 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif

// Host: 2-D bf16 row-major tensor map, box = {64 cols (128 B, SWIZZLE_128B), box_rows}
int br_make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows);
