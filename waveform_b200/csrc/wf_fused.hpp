// wf_fused.hpp — host interface of the fused kernel of the power-of-two sizes (stft_fused_kernel, wf_fused.cuh)
#pragma once
#include "wf_host.hpp"

namespace wf {
// stft_fused_kernel<N, cc, int16 (s16) or float samples> for N = 128 ... 32768, with its CTA size and the shared memory of its
// exchange buffers; *groups := streams per CTA.  A call with display outputs adds the display stage's shared memory.
KernelRef fused_kernel(int N, int cc, bool s16, int *groups);
} // namespace wf
