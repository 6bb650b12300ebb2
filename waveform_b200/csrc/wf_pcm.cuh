// wf_pcm.cuh — the PCM sample formats of wf_batch.pcm_format, as the spectrum kernels' frame loads see them.
//
// Every family loads its frames through Pcm<TS> (TS = float or int16_t): the streamed global loads of one or two samples,
// the read of a sample pair out of a TMA landing buffer, and the byte counts (frame size, TMA transfer, L2 lines).  The
// samples come out as float; an int16 sample v is v * 2^-15, which is exact in float32, so an int16 frame and the float
// frame holding the same values go through the rest of the pipeline (window, FFT, EMA, dB, display) identically.
// Pointers into the PCM stay `const float *` in KParams; Pcm<TS>::base reinterprets them, and offsets count samples.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "wf_fft.cuh"

namespace wf {

__device__ __forceinline__ float2 ldg_stream_f2(const float2 *p)
{
    float2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float ldg_stream_f1(const float *p)
{
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}

template<typename TS>
struct Pcm;

template<>
struct Pcm<float> {
    using Pair = float2;           // two consecutive samples, loaded as one (8-byte aligned)
    static constexpr int kBytes = 4;
    static __host__ __device__ constexpr uint32_t frame_bytes(int n) { return (uint32_t)n * 4u; }
    static __device__ __forceinline__ const float *base(const float *pcm) { return pcm; }
    static __device__ __forceinline__ float load1(const float *q) { return ldg_stream_f1(q); }
    static __device__ __forceinline__ float2 load2(const Pair *q) { return ldg_stream_f2(q); }
    // sample pair n (samples 2n, 2n+1) of a frame staged in shared memory, as a packed complex value
    static __device__ __forceinline__ pk::c64 smem_pair(const void *land, int n)
    {
        return reinterpret_cast<const pk::c64 *>(land)[n];
    }
};

template<>
struct Pcm<int16_t> {
    using Pair = uint32_t;         // two consecutive samples, loaded as one (4-byte aligned)
    static constexpr int kBytes = 2;
    static __host__ __device__ constexpr uint32_t frame_bytes(int n) { return (uint32_t)n * 2u; }
    static __device__ __forceinline__ const int16_t *base(const float *pcm) { return reinterpret_cast<const int16_t *>(pcm); }
    static __device__ __forceinline__ float widen(int v) { return (float)v * 0x1p-15f; }
    static __device__ __forceinline__ float2 widen2(uint32_t w)
    {
        return make_float2(widen((int)(int16_t)(w & 0xffffu)), widen((int)(int16_t)(w >> 16)));
    }
    static __device__ __forceinline__ float load1(const int16_t *q)
    {
        short r;
        asm volatile("ld.global.nc.L1::no_allocate.s16 %0, [%1];" : "=h"(r) : "l"(q));
        return widen(r);
    }
    static __device__ __forceinline__ float2 load2(const Pair *q)
    {
        uint32_t w;
        asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(w) : "l"(q));
        return widen2(w);
    }
    static __device__ __forceinline__ pk::c64 smem_pair(const void *land, int n)
    {
        return pk::from(widen2(reinterpret_cast<const uint32_t *>(land)[n]));
    }
};

} // namespace wf
