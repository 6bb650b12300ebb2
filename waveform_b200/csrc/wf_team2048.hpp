// wf_team2048.hpp — host interface of the team-per-stream N=2048 kernel (wf_team2048.cuh)
#pragma once
#include "wf_host.hpp"

namespace wf {
// stft2048_team_kernel<W, extra, int16 (s16) or float samples> and its CTA size and shared memory.  W = warps per stream (4, 8
// or 16); extra = slope / fast peaks / skip mask / volume / roll-off / peak output in use.  It launches with programmatic
// dependent launch, at most one CTA per SM.
KernelRef team2048_kernel(int W, bool extra, bool s16);
} // namespace wf
