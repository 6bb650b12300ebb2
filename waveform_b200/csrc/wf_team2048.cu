// wf_team2048.cu — instantiations + launcher of stft2048_team_kernel (its own translation unit: compiles in parallel)
#include "wf_host.hpp"
#include "wf_team2048.cuh"
#include "wf_team2048.hpp"

namespace wf {

template<int W, bool EXTRA, typename TS>
static cudaError_t launch(const KParams &kp, int grid, cudaStream_t st, int device)
{
    return launch_kernel(stft2048_team_kernel<W, EXTRA, TS>, device, grid, team::kWarps * 32, team::smem_bytes(), st,
                         {.pdl = true}, kp);
}

template<typename TS>
static cudaError_t launch_w(int W, bool extra, const KParams &kp, int grid, cudaStream_t st, int device)
{
    switch(W)
    {
    case 4: return extra ? launch<4, true, TS>(kp, grid, st, device) : launch<4, false, TS>(kp, grid, st, device);
    case 8: return extra ? launch<8, true, TS>(kp, grid, st, device) : launch<8, false, TS>(kp, grid, st, device);
    case 16: return extra ? launch<16, true, TS>(kp, grid, st, device) : launch<16, false, TS>(kp, grid, st, device);
    default: return cudaErrorInvalidValue;
    }
}

cudaError_t team2048_launch(int W, bool extra, bool s16, const KParams &kp, int grid, cudaStream_t st, int device)
{
    return s16 ? launch_w<int16_t>(W, extra, kp, grid, st, device) : launch_w<float>(W, extra, kp, grid, st, device);
}

} // namespace wf
