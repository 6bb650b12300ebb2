// wf_v3_impl.cuh — the kernel lookup shared by the four instantiation units (wf_v3_c1.cu, wf_v3_c2.cu, wf_v3_s16_c1.cu,
// wf_v3_s16_c2.cu); each compiles it for its own (CC, TS)
#pragma once
#include <cuda_runtime.h>

#include "wf_host.hpp"
#include "wf_v3.cuh"
#include "wf_v3.hpp"

namespace wf {
namespace v3impl {

template<int N, int CC, int EXTRA, typename TS>
KernelRef kernel_r(int R, const KParams &kp, bool display)
{
    const unsigned tn = v3::Geo3<N>::TN;
    const size_t smem = v3::smem_bytes<N>(kp.dch, kp.scratch_q, display, CC, R);
    switch(R)
    {
    case 1:
        if constexpr(N <= 8192)
            return {(const void *)stft_v3_kernel<N, CC, 1, EXTRA, TS>, tn, smem};
        else
            return {};
    case 2: return {(const void *)stft_v3_kernel<N, CC, 2, EXTRA, TS>, tn, smem};
    case 4: return {(const void *)stft_v3_kernel<N, CC, 4, EXTRA, TS>, tn, smem};
    case 8: return {(const void *)stft_v3_kernel<N, CC, 8, EXTRA, TS>, tn, smem};
    default: return {};
    }
}

template<int N, int CC, typename TS>
KernelRef kernel_x(int R, int extra, const KParams &kp, bool display)
{
    return (extra == 0)   ? kernel_r<N, CC, 0, TS>(R, kp, display)
           : (extra == 1) ? kernel_r<N, CC, 1, TS>(R, kp, display)
                          : kernel_r<N, CC, 3, TS>(R, kp, display);
}

} // namespace v3impl

template<int CC, typename TS>
KernelRef v3_kernel(int N, int R, int extra, const KParams &kp, bool display)
{
    switch(N)
    {
    case 1024: return v3impl::kernel_x<1024, CC, TS>(R, extra, kp, display);
    case 2048: return v3impl::kernel_x<2048, CC, TS>(R, extra, kp, display);
    case 4096: return v3impl::kernel_x<4096, CC, TS>(R, extra, kp, display);
    case 8192: return v3impl::kernel_x<8192, CC, TS>(R, extra, kp, display);
    case 16384: return v3impl::kernel_x<16384, CC, TS>(R, extra, kp, display);
    default: return {};
    }
}

} // namespace wf
