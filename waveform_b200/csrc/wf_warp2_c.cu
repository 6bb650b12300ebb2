// wf_warp2_c.cu — stft_warp2_kernel plans, part C: the smaller slider sizes (64-sample steps, src/source.cpp:349)
#include "wf_warp2_impl.cuh"

namespace wf {

Warp2Plan warp2_plan_c(int N)
{
    using namespace warp2;
    switch(N)
    {
        WF_WARP2_CASE(192, 8, 12)
        WF_WARP2_CASE(320, 10, 16)   // also 48 kHz / 144 fps (333 & -16)
        WF_WARP2_CASE(384, 12, 16)
        WF_WARP2_CASE(448, 14, 16)
        WF_WARP2_CASE(576, 16, 18)
        WF_WARP2_CASE(704, 16, 22)
        WF_WARP2_CASE(768, 16, 24)
        WF_WARP2_CASE(832, 16, 26)
        WF_WARP2_CASE(896, 16, 28)
    default: return {};
    }
}

} // namespace wf
