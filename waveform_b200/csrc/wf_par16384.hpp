// wf_par16384.hpp — host interface of the bin-parity cluster kernel for N = 16384 (wf_par16384.cuh)
#pragma once
#include "wf_host.hpp"

namespace wf {
// stft16384_parity_kernel<extra, int16 (s16) or float samples> and its CTA size and shared memory.  It runs one cluster of two
// CTAs per stream and takes the twiddle tables of the N=16384 engine (v3::Tw3 of wf_v3.hpp: tw1 / tw2 of the half-size plan,
// tw0 = W_8192^n of the radix-2 first stage).
KernelRef par16384_kernel(bool extra, bool s16);
} // namespace wf
