// wf_warp2_b.cu — stft_warp2_kernel plans, part B: slider sizes (64-sample steps, src/source.cpp:349)
#include "wf_warp2_impl.cuh"

namespace wf {

Warp2Plan warp2_plan_b(int N)
{
    using namespace warp2;
    switch(N)
    {
        WF_WARP2_CASE(640, 16, 20)
        WF_WARP2_CASE(1152, 24, 24)
        WF_WARP2_CASE(1280, 20, 32)
        WF_WARP2_CASE(1536, 24, 32)
        WF_WARP2_CASE(1792, 28, 32)
        WF_WARP2_CASE(1920, 30, 32)
    default: return {};
    }
}

} // namespace wf
