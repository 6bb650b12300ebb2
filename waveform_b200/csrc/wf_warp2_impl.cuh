// wf_warp2_impl.cuh — plan template shared by the wf_warp2_*.cu instantiation units
#pragma once
#include "wf_host.hpp"
#include "wf_warp2.cuh"
#include "wf_warp2.hpp"

namespace wf {
namespace warp2 {

template<int L, int P>
Warp2Plan plan()
{
    using G = Geo<L, P>;
    return {L, P, G::smem_bytes(0), G::kWarpBytes,
            {{{(const void *)stft_warp2_kernel<L, P, false, false, float>,
               (const void *)stft_warp2_kernel<L, P, false, true, float>},
              {(const void *)stft_warp2_kernel<L, P, true, false, float>,
               (const void *)stft_warp2_kernel<L, P, true, true, float>}},
             {{(const void *)stft_warp2_kernel<L, P, false, false, int16_t>,
               (const void *)stft_warp2_kernel<L, P, false, true, int16_t>},
              {(const void *)stft_warp2_kernel<L, P, true, false, int16_t>,
               (const void *)stft_warp2_kernel<L, P, true, true, int16_t>}}}};
}

#define WF_WARP2_CASE(NN, LL, PP_)                 \
    case NN:                                       \
        static_assert(2 * LL * PP_ == NN, "plan"); \
        return plan<LL, PP_>();

} // namespace warp2
} // namespace wf
