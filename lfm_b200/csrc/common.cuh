// lfm_b200 - sm_90a PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), L2 policies, programmatic dependent launch.
// Hand-written inline PTX; no CUTLASS dependency.  Compile only with
//   -gencode arch=compute_90a,code=sm_90a
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace lfm {

#define LFM_DEVICE __device__ __forceinline__

LFM_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

LFM_DEVICE uint32_t lane_id() {
    uint32_t l;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
    return l;
}

LFM_DEVICE bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// ------------------------------------------------------------------------------------------------
// mbarrier

LFM_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
LFM_DEVICE void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
LFM_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

LFM_DEVICE void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
LFM_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
LFM_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
LFM_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ------------------------------------------------------------------------------------------------
// TMA

LFM_DEVICE void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// 2-D tiled load global -> shared, completion on an mbarrier (transaction bytes).
LFM_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
LFM_DEVICE void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1,
                                 uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
// 2-D tiled store shared -> global (bulk group completion).
LFM_DEVICE void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
LFM_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
LFM_DEVICE void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
LFM_DEVICE void tma_store_wait() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;

// ------------------------------------------------------------------------------------------------
// small math helpers

LFM_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits), .y = hi
    return *reinterpret_cast<uint32_t*>(&h);
}
LFM_DEVICE float tanh_fast(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// GELU(tanh) as in torch.nn.GELU(approximate="tanh")
LFM_DEVICE float gelu_tanh(float x) {
    // 0.5 x (1 + tanh(k0 (x + k1 x^3)))  in 5 FP ops + 1 MUFU:  inner = x (k0 + k0 k1 x^2);  out = hx + hx tanh(inner)
    const float k0 = 0.7978845608028654f, k0k1 = 0.7978845608028654f * 0.044715f;
    const float inner = x * fmaf(k0k1, x * x, k0);
    const float hx = 0.5f * x;
    return fmaf(hx, tanh_fast(inner), hx);
}
LFM_DEVICE float silu(float x) { return x / (1.0f + __expf(-x)); }
// x * rcp.approx(1 + ex2.approx(..)): 5 instructions, 2 of them MUFU, relative error ~2 ulp of fp32 (the result is rounded to bf16).
// The IEEE division above compiles to MUFU.RCP + Newton steps + FCHK + a slow-path call per element, which made the GroupNorm
// apply pass issue-bound at ~60 instructions per element instead of bound by its bytes.
LFM_DEVICE float silu_fast(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

LFM_DEVICE float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
LFM_DEVICE float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// L2 eviction-priority policies for bulk-async (TMA) traffic (the LayerNorm pass's loads of the residual stream with LFM_L2_HINT).
LFM_DEVICE uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
LFM_DEVICE uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may
// start while its predecessor drains; it must not touch global memory the predecessor reads or writes before
// pdl_wait() (which returns once ALL prerequisite grids have completed and flushed).  pdl_trigger() lets the NEXT
// kernel in the stream begin launching.  Both are no-ops for ordinary launches.
LFM_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
LFM_DEVICE void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace lfm
