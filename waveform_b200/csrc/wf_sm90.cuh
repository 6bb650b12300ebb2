// wf_sm90.cuh — the inline-PTX wrappers of the spectrum kernels, one definition each: shared-memory addresses, mbarriers,
// TMA bulk copies and stores, proxy fences, programmatic dependent launch, named and cluster barriers, distributed shared
// memory, streaming stores, the L2 prefetch and the MUFU approximations.  Device code only, no kernels.
// (The PCM loads stay with the sample formats in wf_pcm.cuh, the register packing with the FFT in wf_fft.cuh.)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace wf {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers and TMA bulk copies -----------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// the initialised mbarriers are visible to the async proxy (the TMA engine)
__device__ __forceinline__ void fence_mbarrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted on the mbarrier
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// generic-proxy accesses to shared memory are ordered before later async-proxy (bulk copy) accesses
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// TMA 1-D bulk copy shared -> global, one bulk async-group of the issuing thread per copy
__device__ __forceinline__ void bulk_store_1d(void *dst_gmem, const void *src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// the issuing thread's bulk stores have read their shared-memory source (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// the issuing thread's bulk stores have written global memory, and generic-proxy loads ordered after this see it
__device__ __forceinline__ void bulk_wait_written()
{
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    asm volatile("fence.proxy.async.global;" ::: "memory");
}

// ---- programmatic dependent launch -----------------------------------------------------------------
// the next launch on the stream may start its prologue now
__device__ __forceinline__ void pdl_launch_dependents()
{
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// the previous launch on the stream has completed and its memory operations are visible
__device__ __forceinline__ void pdl_wait()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---- named barrier and thread-block clusters -------------------------------------------------------
// barrier `id` of the CTA for `nthreads` threads (a multiple of 32)
__device__ __forceinline__ void bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ unsigned cluster_ctarank()
{
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// shared::cluster address of the same shared-memory location in the CTA with the given rank
__device__ __forceinline__ uint32_t mapa(uint32_t saddr, unsigned rank)
{
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v)
{
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void st_cluster_u32(uint32_t addr, unsigned v)
{
    asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// ---- global memory: streaming (evict-first) stores, L2 prefetch ------------------------------------
__device__ __forceinline__ void stg_stream(float *p, float v)
{
    asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void stg_stream_v2(float *p, float a, float b)
{
    asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void stg_stream_v4(float *p, float a, float b, float c, float d)
{
    asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// pulls the 128-byte line holding *p into L2
__device__ __forceinline__ void prefetch_l2_line(const void *p)
{
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// ---- MUFU approximations ---------------------------------------------------------------------------
// sqrt.approx.ftz: subnormal inputs and results flush to zero
__device__ __forceinline__ float sqrt_approx_ftz(float x)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// sqrt.approx: subnormal-safe, max relative error 2^-23
__device__ __forceinline__ float sqrt_approx(float x)
{
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// lg2.approx.ftz: log2, -inf below FLT_MIN
__device__ __forceinline__ float lg2_approx_ftz(float x)
{
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

} // namespace wf
