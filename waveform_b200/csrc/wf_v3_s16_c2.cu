// wf_v3_s16_c2.cu — stft_v3_kernel instantiations for int16 samples, two capture channels (separate unit: compiles in parallel)
#include "wf_v3_impl.cuh"

namespace wf {

cudaError_t v3_launch_s16_c2(int N, int R, int extra, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display,
                             int device)
{
    return v3impl::launch_cc<2, int16_t>(N, R, extra, kp, tw, st, display, device);
}

} // namespace wf
