// pattern_probe.cu — bandwidth ceiling of the headline kernel's data movement, without its arithmetic.
// Loaded by tools/pattern_probe.py through ctypes; not part of the product library.
//
//   probe_copy    (a) plain float4 copy: 2 bytes read per byte written, grid-stride
//   probe_stream  (b) the N=2048 warp-per-stream layout of stft2048_fast_kernel: one CTA per SM, W warps, streams dealt
//                     to CTAs then warps, one 8 KiB TMA read per frame into a single landing buffer that is re-requested
//                     halfway through the frame, 32 scalar 4 B stores per lane and row, 4 KiB of state in and out per stream;
//                 (c) as (b), with a separate landing buffer requested a full frame ahead and one 4 KiB cp.async.bulk store
//                     per row from a shared-memory staging row.
// `spin` stands in for the arithmetic: that many SM cycles of busy-wait per frame, split around the (b) re-request.
#include <cstdint>
#include <cuda_runtime.h>

namespace {

constexpr int kN = 2048, kB = 1024;
constexpr int kLand = kN * 4, kRow = kB * 4;
constexpr int kWarpBytes = kLand + kRow + 16;

__device__ __forceinline__ uint32_t su32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile("{\n\t.reg .pred p;\n\tW:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra D;\n\tbra W;\n\tD:\n\t}" ::"r"(su32(bar)),
                 "r"(parity)
                 : "memory");
}

__device__ __forceinline__ void load_frame(void *dst, const float *src, uint64_t *bar)
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su32(bar)), "r"(kLand) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(su32(dst)),
                 "l"(src), "r"(kLand), "r"(su32(bar))
                 : "memory");
}

__device__ __forceinline__ void spin_for(int cycles)
{
    if(cycles <= 0)
        return;
    const long long c0 = clock64();
    while(clock64() - c0 < cycles)
        ;
}

__global__ void probe_copy_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, long long n_out)
{
    for(long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_out; i += (long long)gridDim.x * blockDim.x)
    {
        const float4 a = __ldcs(in + 2 * i), b = __ldcs(in + 2 * i + 1);
        __stcs(out + i, make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w));
    }
}

template<bool FULL_LEAD_BULK>
__global__ void __launch_bounds__(16 * 32, 1) probe_stream_kernel(const float *pcm, float *out, float *state, int S, int T, int spin)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5, G = gridDim.x;
    unsigned char *wb = smem + warp * kWarpBytes;
    const float2 *land = reinterpret_cast<const float2 *>(wb);
    float *row = reinterpret_cast<float *>(wb + kLand);
    uint64_t *bar = reinterpret_cast<uint64_t *>(wb + kLand + kRow);
    if(lane == 0)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(su32(bar)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const int n_local = (S > (int)blockIdx.x) ? (S - (int)blockIdx.x + G - 1) / G : 0;
    const int nseg = (n_local > warp) ? (n_local - warp + W - 1) / W : 0;
    // the same bin pairs as the kernel: k1 = lane + 32 q, k2 = kb + 32 (31 - q), lane 0's first pair (0, 512)
    const int kb = ((32 - lane) & 31) + (lane == 0 ? 32 : 0);
    const int k2_q0 = (lane == 0) ? 512 : (kb + 992);
    uint32_t phase = 0;
    if(nseg > 0 && lane == 0)
        load_frame(wb, pcm + (size_t)(blockIdx.x + warp * G) * T * kN, bar);
    for(int j = 0; j < nseg; ++j)
    {
        const int s = (int)blockIdx.x + (warp + j * W) * G;
        const int s_next = (j + 1 < nseg) ? s + W * G : -1;
        float acc = 0.0f;
        for(int q = 0; q < 32; ++q)
            acc += state[(size_t)s * kB + lane + 32 * q];
        for(int t = 0; t < T; ++t)
        {
            const float *next = (t + 1 < T) ? pcm + ((size_t)s * T + t + 1) * kN : (s_next >= 0 ? pcm + (size_t)s_next * T * kN : nullptr);
            mbar_wait(bar, phase);
            phase ^= 1u;
#pragma unroll
            for(int i = 0; i < 32; ++i)
            {
                const float2 v = land[lane + 32 * i];
                acc += v.x + v.y;
            }
            __syncwarp();
            if(FULL_LEAD_BULK && lane == 0 && next != nullptr)
                load_frame(wb, next, bar);
            spin_for(FULL_LEAD_BULK ? spin : spin / 2);
            if(!FULL_LEAD_BULK && lane == 0 && next != nullptr)
                load_frame(wb, next, bar);
            spin_for(FULL_LEAD_BULK ? 0 : spin - spin / 2);
            float *orow = out + ((size_t)s * T + t) * kB;
            if(FULL_LEAD_BULK)
            {
                if(lane == 0)
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                __syncwarp();
            }
#pragma unroll
            for(int q = 0; q < 16; ++q)
            {
                const int k1 = lane + 32 * q, k2 = (q == 0) ? k2_q0 : (kb + 32 * (31 - q));
                if(FULL_LEAD_BULK)
                {
                    row[k1] = acc;
                    row[k2] = acc;
                }
                else
                {
                    __stcs(orow + k1, acc);
                    __stcs(orow + k2, acc);
                }
            }
            if(FULL_LEAD_BULK)
            {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if(lane == 0)
                {
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(orow), "r"(su32(row)), "r"(kRow)
                                 : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        for(int q = 0; q < 32; ++q)
            state[(size_t)s * kB + lane + 32 * q] = acc;
    }
    if(FULL_LEAD_BULK && lane == 0)
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

} // namespace

// Each entry point runs `iters` launches after `warmup` and returns milliseconds per launch (CUDA events), < 0 on error.
extern "C" float probe_copy(const float *in, float *out, long long n_out_floats, int blocks, int threads, int warmup, int iters)
{
    auto go = [&] { probe_copy_kernel<<<blocks, threads>>>(reinterpret_cast<const float4 *>(in), reinterpret_cast<float4 *>(out), n_out_floats / 4); };
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for(int i = 0; i < warmup; ++i)
        go();
    cudaEventRecord(e0);
    for(int i = 0; i < iters; ++i)
        go();
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = -1.0f;
    if(cudaGetLastError() == cudaSuccess)
        cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return ms < 0 ? ms : ms / iters;
}

extern "C" float probe_stream(int full_lead_bulk, const float *pcm, float *out, float *state, int S, int T, int sms, int warps,
                              int spin, int warmup, int iters)
{
    const int grid = S < sms ? S : sms;
    const size_t smem = (size_t)warps * kWarpBytes;
    auto kern = full_lead_bulk ? probe_stream_kernel<true> : probe_stream_kernel<false>;
    if(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return -1.0f;
    auto go = [&] { kern<<<grid, warps * 32, smem>>>(pcm, out, state, S, T, spin); };
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for(int i = 0; i < warmup; ++i)
        go();
    cudaEventRecord(e0);
    for(int i = 0; i < iters; ++i)
        go();
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = -1.0f;
    if(cudaGetLastError() == cudaSuccess)
        cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return ms < 0 ? ms : ms / iters;
}
