// wf_v3_s16_c2.cu — stft_v3_kernel instantiations for int16 samples, two capture channels (separate unit: compiles in parallel)
#include "wf_v3_impl.cuh"

namespace wf {

template KernelRef v3_kernel<2, int16_t>(int N, int R, int extra, const KParams &kp, bool display);

} // namespace wf
