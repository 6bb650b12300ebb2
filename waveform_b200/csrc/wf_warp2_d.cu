// wf_warp2_d.cu — stft_warp2_kernel plans, part D: the larger slider sizes and more automatic sizes (sr/fps & -16)
#include "wf_warp2_impl.cuh"

namespace wf {

Warp2Plan warp2_plan_d(int N)
{
    using namespace warp2;
    switch(N)
    {
        WF_WARP2_CASE(1344, 24, 28)
        WF_WARP2_CASE(1408, 22, 32)
        WF_WARP2_CASE(1664, 26, 32)
        WF_WARP2_CASE(1728, 27, 32)
        WF_WARP2_CASE(880, 20, 22)   // 44.1 kHz / 50 fps (882 & -16)
        WF_WARP2_CASE(480, 15, 16)   // 48 kHz / 100 fps
        WF_WARP2_CASE(528, 12, 22)   // 48 kHz / 90 fps (533 & -16)
        WF_WARP2_CASE(352, 11, 16)   // 44.1 kHz / 120 fps (367 & -16)
        WF_WARP2_CASE(288, 12, 12)   // 48 kHz / 165 fps (290 & -16)
    default: return {};
    }
}

} // namespace wf
