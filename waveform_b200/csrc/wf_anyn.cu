// wf_anyn.cu — instantiations of stft_anyn_kernel (its own translation unit)
#include "wf_host.hpp"
#include "wf_anyn.cuh"
#include "wf_anyn.hpp"

namespace wf {

KernelRef anyn_kernel(int cc, bool s16)
{
    const void *const kernels[2][2] = {
        {(const void *)stft_anyn_kernel<1, float>, (const void *)stft_anyn_kernel<2, float>},
        {(const void *)stft_anyn_kernel<1, int16_t>, (const void *)stft_anyn_kernel<2, int16_t>}};
    return {kernels[s16][cc - 1], kAnyThreads, 0};
}

} // namespace wf
