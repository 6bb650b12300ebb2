// wf_warp2_e.cu — stft_warp2_kernel plans, part E: power-of-two sizes.  Used for DISPLAY outputs of one-channel sources
// (curve points / bars / pixels: BASELINE config 1 = N 1024 with 26 bars): the spectrum-only N=2048 path is wf_fast2048.cuh and
// the other spectrum-only power-of-two sizes stay on the CTA-per-tick kernel (wf_v3.cuh).
#include "wf_warp2_impl.cuh"

namespace wf {

Warp2Plan warp2_plan_e(int N)
{
    using namespace warp2;
    switch(N)
    {
        WF_WARP2_CASE(512, 16, 16)
        WF_WARP2_CASE(1024, 16, 32)  // 32 lanes in pass B and in the epilogue (8 bin pairs per lane)
        WF_WARP2_CASE(2048, 32, 32)
    default: return {};
    }
}

} // namespace wf
