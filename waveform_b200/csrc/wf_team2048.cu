// wf_team2048.cu — instantiations of stft2048_team_kernel (its own translation unit: compiles in parallel)
#include "wf_host.hpp"
#include "wf_team2048.cuh"
#include "wf_team2048.hpp"

namespace wf {

template<int W, typename TS>
static const void *kernel(bool extra)
{
    return extra ? (const void *)stft2048_team_kernel<W, true, TS> : (const void *)stft2048_team_kernel<W, false, TS>;
}

template<typename TS>
static const void *kernel_w(int W, bool extra)
{
    switch(W)
    {
    case 4: return kernel<4, TS>(extra);
    case 8: return kernel<8, TS>(extra);
    case 16: return kernel<16, TS>(extra);
    default: return nullptr;
    }
}

KernelRef team2048_kernel(int W, bool extra, bool s16)
{
    return {s16 ? kernel_w<int16_t>(W, extra) : kernel_w<float>(W, extra), team::kWarps * 32, team::smem_bytes()};
}

} // namespace wf
