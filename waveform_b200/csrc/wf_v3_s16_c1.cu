// wf_v3_s16_c1.cu — stft_v3_kernel instantiations for int16 samples, one capture channel (separate unit: compiles in parallel)
#include "wf_v3_impl.cuh"

namespace wf {

cudaError_t v3_launch_s16_c2(int N, int R, int extra, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display,
                             int device);

cudaError_t v3_launch_s16(int N, int cc, int R, int extra, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display,
                          int device)
{
    if(cc == 2)
        return v3_launch_s16_c2(N, R, extra, kp, tw, st, display, device);
    return v3impl::launch_cc<1, int16_t>(N, R, extra, kp, tw, st, display, device);
}

} // namespace wf
