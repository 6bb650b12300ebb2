// wf_team2048.hpp — host interface of the team-per-stream N=2048 kernel (wf_team2048.cuh)
#pragma once
#include <cuda_runtime.h>

namespace wf {
struct KParams;
// W = warps per stream (4, 8 or 16); grid = CTAs (one per SM at most); extra = slope / fast peaks / skip mask / volume /
// roll-off / peak output in use; s16 = int16 samples.  Launches with programmatic dependent launch.
cudaError_t team2048_launch(int W, bool extra, bool s16, const KParams &kp, int grid, cudaStream_t st, int device);
} // namespace wf
