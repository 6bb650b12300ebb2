// wf_warp2_impl.cuh — launcher template shared by the wf_warp2_*.cu instantiation units
#pragma once
#include "wf_warp2.cuh"
#include "wf_warp2.hpp"

namespace wf {
namespace warp2 {

constexpr int kMaxSmem = 227 * 1024; // opt-in shared memory per CTA on sm_90

template<int L, int P, bool EXTRA, bool DISP>
cudaError_t launch(const KParams &kp, int grid, int *warps_io, cudaStream_t st, bool pdl, int device)
{
    using G = Geo<L, P>;
    static thread_local bool configured[64] = {false};
    const int dev = device & 63;
    if(!configured[dev])
    {
        cudaError_t err = cudaFuncSetAttribute(stft_warp2_kernel<L, P, EXTRA, DISP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               DISP ? kMaxSmem : G::smem_bytes(G::kWarps));
        if(err != cudaSuccess)
            return err;
        configured[dev] = true;
    }
    int warps = *warps_io;
    const size_t per_warp_extra = DISP ? (size_t)kp.disp_bytes : 0, cta_extra = DISP ? (size_t)kp.disp_tab_bytes : 0;
    while(warps > 1 && G::smem_bytes(warps) + cta_extra + warps * per_warp_extra > (size_t)kMaxSmem)
        --warps; // the display rows cost warps per SM at the largest sizes; the streams simply take more rounds
    if(G::smem_bytes(warps) + cta_extra + warps * per_warp_extra > (size_t)kMaxSmem)
        return cudaErrorInvalidConfiguration;
    *warps_io = warps;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)(warps * 32));
    cfg.dynamicSmemBytes = G::smem_bytes(warps) + cta_extra + warps * per_warp_extra;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, stft_warp2_kernel<L, P, EXTRA, DISP>, kp);
}

#define WF_WARP2_CASE(NN, LL, PP_)                                                                                       \
    case NN:                                                                                                             \
        static_assert(2 * LL * PP_ == NN, "plan");                                                                      \
        *name = disp ? "stft_warp2_kernel<" #LL "," #PP_ ",display>" : "stft_warp2_kernel<" #LL "," #PP_ ">";          \
        if(disp)                                                                                                         \
            return extra ? launch<LL, PP_, true, true>(kp, grid, warps, st, pdl, device)                                 \
                         : launch<LL, PP_, false, true>(kp, grid, warps, st, pdl, device);                               \
        return extra ? launch<LL, PP_, true, false>(kp, grid, warps, st, pdl, device)                                    \
                     : launch<LL, PP_, false, false>(kp, grid, warps, st, pdl, device);

} // namespace warp2
} // namespace wf
