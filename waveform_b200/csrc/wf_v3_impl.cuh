// wf_v3_impl.cuh — launcher template shared by the two instantiation units (wf_v3_c1.cu / wf_v3_c2.cu)
#pragma once
#include <cuda_runtime.h>

#include "wf_host.hpp"
#include "wf_v3.cuh"
#include "wf_v3.hpp"

namespace wf {
namespace v3impl {

template<int N, int CC, int R, int EXTRA, typename TS>
cudaError_t launch_one(const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display, int device)
{
    return launch_kernel(stft_v3_kernel<N, CC, R, EXTRA, TS>, device, kp.n_streams * R, v3::Geo3<N>::TN,
                         v3::smem_bytes<N>(kp.dch, kp.scratch_q, display, CC, R), st, {.cluster = R}, kp, tw);
}

template<int N, int CC, int EXTRA, typename TS>
cudaError_t launch_r(int R, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display, int device)
{
    switch(R)
    {
    case 1:
        if constexpr(N <= 8192)
            return launch_one<N, CC, 1, EXTRA, TS>(kp, tw, st, display, device);
        else
            return cudaErrorInvalidValue;
    case 2: return launch_one<N, CC, 2, EXTRA, TS>(kp, tw, st, display, device);
    case 4: return launch_one<N, CC, 4, EXTRA, TS>(kp, tw, st, display, device);
    case 8: return launch_one<N, CC, 8, EXTRA, TS>(kp, tw, st, display, device);
    default: return cudaErrorInvalidValue;
    }
}

template<int CC, typename TS>
cudaError_t launch_cc(int N, int R, int extra, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display, int device)
{
    switch(N)
    {
    case 1024:
        return (extra == 0)   ? launch_r<1024, CC, 0, TS>(R, kp, tw, st, display, device)
               : (extra == 1) ? launch_r<1024, CC, 1, TS>(R, kp, tw, st, display, device)
                              : launch_r<1024, CC, 3, TS>(R, kp, tw, st, display, device);
    case 2048:
        return (extra == 0)   ? launch_r<2048, CC, 0, TS>(R, kp, tw, st, display, device)
               : (extra == 1) ? launch_r<2048, CC, 1, TS>(R, kp, tw, st, display, device)
                              : launch_r<2048, CC, 3, TS>(R, kp, tw, st, display, device);
    case 4096:
        return (extra == 0)   ? launch_r<4096, CC, 0, TS>(R, kp, tw, st, display, device)
               : (extra == 1) ? launch_r<4096, CC, 1, TS>(R, kp, tw, st, display, device)
                              : launch_r<4096, CC, 3, TS>(R, kp, tw, st, display, device);
    case 8192:
        return (extra == 0)   ? launch_r<8192, CC, 0, TS>(R, kp, tw, st, display, device)
               : (extra == 1) ? launch_r<8192, CC, 1, TS>(R, kp, tw, st, display, device)
                              : launch_r<8192, CC, 3, TS>(R, kp, tw, st, display, device);
    case 16384:
        return (extra == 0)   ? launch_r<16384, CC, 0, TS>(R, kp, tw, st, display, device)
               : (extra == 1) ? launch_r<16384, CC, 1, TS>(R, kp, tw, st, display, device)
                              : launch_r<16384, CC, 3, TS>(R, kp, tw, st, display, device);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace v3impl
} // namespace wf
