// wf_warp2_a.cu — stft_warp2_kernel plans, part A: the automatic sizes sr/fps & -16 (src/source.cpp:1161-1167)
#include "wf_warp2_impl.cuh"

namespace wf {

Warp2Plan warp2_plan_b(int N);
Warp2Plan warp2_plan_c(int N);
Warp2Plan warp2_plan_d(int N);
Warp2Plan warp2_plan_e(int N);

Warp2Plan warp2_plan(int N)
{
    using namespace warp2;
    switch(N)
    {
        WF_WARP2_CASE(400, 10, 20)   // 48 kHz / 120 fps
        WF_WARP2_CASE(720, 18, 20)   // 44.1 kHz / 60 fps (735 & -16)
        WF_WARP2_CASE(800, 20, 20)   // 48 kHz / 60 fps: the plugin's default configuration
        WF_WARP2_CASE(960, 20, 24)   // 48 kHz / 50 fps
        WF_WARP2_CASE(1456, 26, 28)  // 44.1 kHz / 30 fps (1470 & -16): 2^4 7 13
        WF_WARP2_CASE(1600, 25, 32)  // 48 kHz / 30 fps
    default: break;
    }
    for(auto part : {warp2_plan_b, warp2_plan_c, warp2_plan_d, warp2_plan_e})
        if(const Warp2Plan p = part(N); p.L)
            return p;
    return {};
}

} // namespace wf
