// wf_par16384.cu — instantiations + launcher of stft16384_parity_kernel (its own translation unit)
#include "wf_host.hpp"
#include "wf_par16384.cuh"
#include "wf_par16384.hpp"

namespace wf {

template<bool EXTRA, typename TS>
static cudaError_t launch(const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, int device)
{
    return launch_kernel(stft16384_parity_kernel<EXTRA, TS>, device, 2 * kp.n_streams, par16384::kTN, par16384::smem_bytes(),
                         st, {}, kp, tw);
}

cudaError_t par16384_launch(bool extra, bool s16, const KParams &kp, const float *d_tw1, const float *d_tw2, const float *d_tw0,
                            cudaStream_t st, int device)
{
    v3::Tw3 tw{reinterpret_cast<const float2 *>(d_tw1), reinterpret_cast<const float2 *>(d_tw2),
               reinterpret_cast<const float2 *>(d_tw0)};
    if(s16)
        return extra ? launch<true, int16_t>(kp, tw, st, device) : launch<false, int16_t>(kp, tw, st, device);
    return extra ? launch<true, float>(kp, tw, st, device) : launch<false, float>(kp, tw, st, device);
}

} // namespace wf
