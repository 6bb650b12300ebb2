// wf_team2048.cu — instantiations + launcher of stft2048_team_kernel (its own translation unit: compiles in parallel)
#include "wf_host.hpp"
#include "wf_team2048.cuh"
#include "wf_team2048.hpp"

namespace wf {

template<int W, bool EXTRA>
static cudaError_t launch(const KParams &kp, int grid, cudaStream_t st, int device)
{
    return launch_kernel(stft2048_team_kernel<W, EXTRA>, device, grid, team::kWarps * 32, team::smem_bytes(), st,
                         {.pdl = true}, kp);
}

cudaError_t team2048_launch(int W, bool extra, const KParams &kp, int grid, cudaStream_t st, int device)
{
    switch(W)
    {
    case 4: return extra ? launch<4, true>(kp, grid, st, device) : launch<4, false>(kp, grid, st, device);
    case 8: return extra ? launch<8, true>(kp, grid, st, device) : launch<8, false>(kp, grid, st, device);
    case 16: return extra ? launch<16, true>(kp, grid, st, device) : launch<16, false>(kp, grid, st, device);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace wf
