// wf_wide.cu — instantiations + launcher of the cluster kernel (wf_wide.cuh); a separate translation unit so that it
// compiles in parallel with wf_engine.cu.
#include <cuda_runtime.h>

#include "wf_host.hpp"
#include "wf_wide.cuh"
#include "wf_wide.hpp"

namespace wf {

namespace {

template<int N, int CC, int R, typename TS>
cudaError_t launch_one(const KParams &kp, cudaStream_t st, bool display, int device)
{
    return launch_kernel(stft_wide_kernel<N, CC, R, TS>, device, kp.n_streams * R, Geo<N>::TN,
                         wide::smem_bytes<N>(kp.dch, kp.scratch_q, display), st, {.cluster = R}, kp);
}

template<int N, int CC, typename TS>
cudaError_t launch_r(int R, const KParams &kp, cudaStream_t st, bool display, int device)
{
    switch(R)
    {
    case 2: return launch_one<N, CC, 2, TS>(kp, st, display, device);
    case 4: return launch_one<N, CC, 4, TS>(kp, st, display, device);
    case 8: return launch_one<N, CC, 8, TS>(kp, st, display, device);
    default: return cudaErrorInvalidValue;
    }
}

template<int CC, typename TS>
cudaError_t launch_n(int N, int R, const KParams &kp, cudaStream_t st, bool display, int device)
{
    switch(N)
    {
    case 4096: return launch_r<4096, CC, TS>(R, kp, st, display, device);
    case 8192: return launch_r<8192, CC, TS>(R, kp, st, display, device);
    case 16384: return launch_r<16384, CC, TS>(R, kp, st, display, device);
    case 32768: return launch_r<32768, CC, TS>(R, kp, st, display, device);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace

bool wide_supported(int N) { return N == 4096 || N == 8192 || N == 16384 || N == 32768; }

size_t wide_smem_bytes(int N, int dch, int n_points, bool display)
{
    switch(N)
    {
    case 4096: return wide::smem_bytes<4096>(dch, n_points, display);
    case 8192: return wide::smem_bytes<8192>(dch, n_points, display);
    case 16384: return wide::smem_bytes<16384>(dch, n_points, display);
    case 32768: return wide::smem_bytes<32768>(dch, n_points, display);
    default: return 0;
    }
}

cudaError_t wide_launch(int N, int cc, int R, bool s16, const KParams &kp, cudaStream_t st, bool display, int device)
{
    if(s16)
        return (cc == 2) ? launch_n<2, int16_t>(N, R, kp, st, display, device) : launch_n<1, int16_t>(N, R, kp, st, display, device);
    return (cc == 2) ? launch_n<2, float>(N, R, kp, st, display, device) : launch_n<1, float>(N, R, kp, st, display, device);
}

} // namespace wf
