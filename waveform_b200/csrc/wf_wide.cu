// wf_wide.cu — instantiations of the cluster kernel (wf_wide.cuh); a separate translation unit so that it compiles in
// parallel with wf_engine.cu.
#include <cuda_runtime.h>

#include "wf_host.hpp"
#include "wf_wide.cuh"
#include "wf_wide.hpp"

namespace wf {

namespace {

template<int N, int CC, typename TS>
KernelRef kernel_r(int R, const KParams &kp, bool display)
{
    const size_t smem = wide::smem_bytes<N>(kp.dch, kp.scratch_q, display);
    switch(R)
    {
    case 2: return {(const void *)stft_wide_kernel<N, CC, 2, TS>, Geo<N>::TN, smem};
    case 4: return {(const void *)stft_wide_kernel<N, CC, 4, TS>, Geo<N>::TN, smem};
    case 8: return {(const void *)stft_wide_kernel<N, CC, 8, TS>, Geo<N>::TN, smem};
    default: return {};
    }
}

template<int CC, typename TS>
KernelRef kernel_n(int N, int R, const KParams &kp, bool display)
{
    switch(N)
    {
    case 4096: return kernel_r<4096, CC, TS>(R, kp, display);
    case 8192: return kernel_r<8192, CC, TS>(R, kp, display);
    case 16384: return kernel_r<16384, CC, TS>(R, kp, display);
    case 32768: return kernel_r<32768, CC, TS>(R, kp, display);
    default: return {};
    }
}

} // namespace

KernelRef wide_kernel(int N, int cc, int R, bool s16, const KParams &kp, bool display)
{
    if(s16)
        return (cc == 2) ? kernel_n<2, int16_t>(N, R, kp, display) : kernel_n<1, int16_t>(N, R, kp, display);
    return (cc == 2) ? kernel_n<2, float>(N, R, kp, display) : kernel_n<1, float>(N, R, kp, display);
}

} // namespace wf
