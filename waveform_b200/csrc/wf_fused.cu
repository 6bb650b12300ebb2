// wf_fused.cu — instantiations of stft_fused_kernel (its own translation unit)
#include "wf_host.hpp"
#include "wf_fused.hpp"
#include "wf_fused.cuh"

namespace wf {

template<int N, int CC, typename TS>
static KernelRef kernel(int *groups)
{
    using G = Geo<N>;
    *groups = G::GROUPS;
    return {(const void *)stft_fused_kernel<N, CC, TS>, G::CTA, (size_t)G::GROUPS * G::BUF * sizeof(float2)};
}

template<int CC, typename TS>
static KernelRef kernel_n(int N, int *groups)
{
    switch(N)
    {
    case 128: return kernel<128, CC, TS>(groups);
    case 256: return kernel<256, CC, TS>(groups);
    case 512: return kernel<512, CC, TS>(groups);
    case 1024: return kernel<1024, CC, TS>(groups);
    case 2048: return kernel<2048, CC, TS>(groups);
    case 4096: return kernel<4096, CC, TS>(groups);
    case 8192: return kernel<8192, CC, TS>(groups);
    case 16384: return kernel<16384, CC, TS>(groups);
    case 32768: return kernel<32768, CC, TS>(groups);
    default: return {};
    }
}

KernelRef fused_kernel(int N, int cc, bool s16, int *groups)
{
    if(s16)
        return (cc == 2) ? kernel_n<2, int16_t>(N, groups) : kernel_n<1, int16_t>(N, groups);
    return (cc == 2) ? kernel_n<2, float>(N, groups) : kernel_n<1, float>(N, groups);
}

} // namespace wf
