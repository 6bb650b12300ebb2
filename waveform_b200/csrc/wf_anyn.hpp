// wf_anyn.hpp — host interface of the any-N kernel (wf_anyn.cuh): its run-time FFT plan, its CTA size and the lookup of its
// instantiations (wf_anyn.cu)
#pragma once
#include <cuda_runtime.h>

#include "wf_host.hpp"

namespace wf {

struct AnyPlan {
    int M;          // N/2
    int n_pass;
    int radix[20];
    float2 *scratch; // per-CTA [2][M] complex work buffers in global memory (L2) when they do not fit in shared
                     // memory (N > ~27000, e.g. the plugin's "large FFT" sizes up to 65536); null = shared memory
};

constexpr int kAnyThreads = 256;

// stft_anyn_kernel<cc, int16 (s16) or float samples> with its kAnyThreads threads per CTA.  Its dynamic shared memory
// depends on the call (work buffers and display rows), so smem is 0 here.  It takes the call's AnyPlan after KParams.
KernelRef anyn_kernel(int cc, bool s16);

} // namespace wf
