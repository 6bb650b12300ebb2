// wf_warp2_impl.cuh — plan template shared by the wf_warp2_*.cu instantiation units
#pragma once
#include "wf_host.hpp"
#include "wf_warp2.cuh"
#include "wf_warp2.hpp"

namespace wf {
namespace warp2 {

template<int L, int P, bool EXTRA, bool DISP, typename TS>
cudaError_t launch(const KParams &kp, int grid, int warps, size_t smem, cudaStream_t st, int device)
{
    return launch_kernel(stft_warp2_kernel<L, P, EXTRA, DISP, TS>, device, grid, warps * 32, smem, st, {.pdl = true}, kp);
}

template<int L, int P>
Warp2Plan plan()
{
    using G = Geo<L, P>;
    return {L, P, G::smem_bytes(0), G::kWarpBytes,
            {{{launch<L, P, false, false, float>, launch<L, P, false, true, float>},
              {launch<L, P, true, false, float>, launch<L, P, true, true, float>}},
             {{launch<L, P, false, false, int16_t>, launch<L, P, false, true, int16_t>},
              {launch<L, P, true, false, int16_t>, launch<L, P, true, true, int16_t>}}}};
}

#define WF_WARP2_CASE(NN, LL, PP_)                 \
    case NN:                                       \
        static_assert(2 * LL * PP_ == NN, "plan"); \
        return plan<LL, PP_>();

} // namespace warp2
} // namespace wf
