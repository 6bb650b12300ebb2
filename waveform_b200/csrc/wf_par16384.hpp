// wf_par16384.hpp — host interface of the bin-parity cluster kernel for N = 16384 (wf_par16384.cuh)
#pragma once
#include <cuda_runtime.h>

namespace wf {
struct KParams;
// one cluster of two CTAs per stream; the twiddle tables are those of the N=16384 engine (wf_v3.hpp: tw1 / tw2 of the
// half-size plan, tw0 = W_8192^n of the radix-2 first stage); s16 = int16 samples
cudaError_t par16384_launch(bool extra, bool s16, const KParams &kp, const float *d_tw1, const float *d_tw2, const float *d_tw0,
                            cudaStream_t st, int device);
} // namespace wf
