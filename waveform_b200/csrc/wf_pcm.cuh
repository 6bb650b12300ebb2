// wf_pcm.cuh — the PCM sample formats (wf_pcm_format) of wf_batch, wf_meter_batch and wf_wave_batch, as the kernels of all
// three engines load them.
//
// Every kernel that reads PCM does so through Pcm<TS> (TS = float or int16_t).  The spectrum families use the streamed
// global loads of one or two samples, the read of a sample pair out of a TMA landing buffer, and the byte counts (frame size,
// TMA transfer, L2 lines).  The level meter uses the read-only-path loads of one sample and of a group of four (16 bytes of
// float, 8 bytes of int16), and the waveform gathers single samples.  The samples come out as float; an int16 sample v is
// v * 2^-15, which is exact in float32, so int16 input and the float input holding the same values go through the rest of
// each pipeline (window, FFT, EMA, dB, display; the meter's sums and ring; the waveform's buffers) identically.
// Pointers into the PCM stay `const float *` in the kernels' parameters; Pcm<TS>::base reinterprets them, and offsets
// count samples.
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
    using Quad = float4;           // four consecutive samples, loaded as one (16-byte aligned)
    static constexpr int kBytes = 4;
    static __host__ __device__ constexpr uint32_t frame_bytes(int n) { return (uint32_t)n * 4u; }
    static __device__ __forceinline__ const float *base(const float *pcm) { return pcm; }
    static __device__ __forceinline__ float load1(const float *q) { return ldg_stream_f1(q); }
    static __device__ __forceinline__ float2 load2(const Pair *q) { return ldg_stream_f2(q); }
    // read-only-path loads (ld.global.nc) of one sample and of four
    static __device__ __forceinline__ float ldg1(const float *q) { return __ldg(q); }
    static __device__ __forceinline__ float4 ldg4(const Quad *q) { return __ldg(q); }
    // sample pair n (samples 2n, 2n+1) of a frame staged in shared memory, as a packed complex value
    static __device__ __forceinline__ pk::c64 smem_pair(const void *land, int n)
    {
        return reinterpret_cast<const pk::c64 *>(land)[n];
    }
};

template<>
struct Pcm<int16_t> {
    using Pair = uint32_t;         // two consecutive samples, loaded as one (4-byte aligned)
    using Quad = uint2;            // four consecutive samples, loaded as one (8-byte aligned)
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
    // The same value as widen(): the bits 0x4b400000 + v are the float 1.5 * 2^23 + v (its ulp is 1), and
    // (1.5 * 2^23 + v) * 2^-15 - 384 = v * 2^-15 is exact in one FMA (v = 0 gives +0.0f).  An integer add and an FMA in
    // place of I2F keep the waveform display kernels within their 64 registers without spills.
    static __device__ __forceinline__ float ldg1(const int16_t *q)
    {
        return __fmaf_rn(__int_as_float(0x4b400000 + (int)__ldg(q)), 0x1p-15f, -384.0f);
    }
    static __device__ __forceinline__ float4 ldg4(const Quad *q) // widened in sample order
    {
        const uint2 w = __ldg(q);
        const float2 lo = widen2(w.x), hi = widen2(w.y);
        return make_float4(lo.x, lo.y, hi.x, hi.y);
    }
    static __device__ __forceinline__ pk::c64 smem_pair(const void *land, int n)
    {
        return pk::from(widen2(reinterpret_cast<const uint32_t *>(land)[n]));
    }
};

} // namespace wf
