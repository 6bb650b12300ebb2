// wf_wide.hpp — host interface of the cluster kernel (wf_wide.cuh / wf_wide.cu)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "wf_host.hpp"

namespace wf {
struct KParams;
// stft_wide_kernel<N, cc, R, int16 (s16) or float samples> with its threads per CTA and its shared memory at kp's display
// settings (dch, scratch_q); R = cluster size (2, 4 or 8 CTAs per stream)
KernelRef wide_kernel(int N, int cc, int R, bool s16, const KParams &kp, bool display);
} // namespace wf
