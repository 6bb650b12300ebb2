// wf_par16384.cu — instantiations of stft16384_parity_kernel (its own translation unit)
#include "wf_host.hpp"
#include "wf_par16384.cuh"
#include "wf_par16384.hpp"

namespace wf {

KernelRef par16384_kernel(bool extra, bool s16)
{
    const void *const kernels[2][2] = {
        {(const void *)stft16384_parity_kernel<false, float>, (const void *)stft16384_parity_kernel<true, float>},
        {(const void *)stft16384_parity_kernel<false, int16_t>, (const void *)stft16384_parity_kernel<true, int16_t>}};
    return {kernels[s16][extra], par16384::kTN, par16384::smem_bytes()};
}

} // namespace wf
