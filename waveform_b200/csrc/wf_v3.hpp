// wf_v3.hpp — host interface of the CTA-per-tick kernel for fft sizes 4096 / 8192 / 16384 (wf_v3.cuh)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <vector>

#include "wf_host.hpp"

namespace wf {
struct KParams;
namespace v3 {
// the inter-pass twiddle tables (v3_build_twiddles) as the CTA-per-tick and N=16384 parity kernels take them after KParams
struct Tw3 {
    const float2 *tw1; // [A][TN]  W_M^(t*ka)
    const float2 *tw2; // [B][C]   W_(B*C)^(c*kb)
    const float2 *tw0; // split plan only: [16][TN] W_M^(a*TN + t) of the radix-2 first stage (tw1/tw2 are the half size's)
};
} // namespace v3
int v3_min_cluster(int N); // smallest supported cluster size (1, or 2 where the per-thread state would not fit registers)
// Inter-pass twiddle tables (interleaved re,im), evaluated in double: tw1[ka][t] = W_M^(t*ka), tw2[kb][c] = W_(BC)^(c*kb);
// tw0 (16384 only) = W_M^(a*TN + t) of the radix-2 first stage, tw1/tw2 then belong to the 4096-point sub-FFTs.  All three
// stay empty for sizes without the kernel.
void v3_build_twiddles(int N, std::vector<float> &tw1, std::vector<float> &tw2, std::vector<float> &tw0);
// stft_v3_kernel<N, CC, R, EXTRA, TS> with its threads per CTA and its shared memory at kp's display settings (dch,
// scratch_q).  R = CTAs per stream (1 = no cluster); extra: 0 = plain, 1 = per-tick peak output only, 3 = slope / fast peaks
// / skip mask / volume / roll-off in use (with or without the peak output).  Each wf_v3_*.cu unit compiles one (CC, TS).
template<int CC, typename TS>
KernelRef v3_kernel(int N, int R, int extra, const KParams &kp, bool display);
extern template KernelRef v3_kernel<1, float>(int, int, int, const KParams &, bool);   // wf_v3_c1.cu
extern template KernelRef v3_kernel<2, float>(int, int, int, const KParams &, bool);   // wf_v3_c2.cu
extern template KernelRef v3_kernel<1, int16_t>(int, int, int, const KParams &, bool); // wf_v3_s16_c1.cu
extern template KernelRef v3_kernel<2, int16_t>(int, int, int, const KParams &, bool); // wf_v3_s16_c2.cu
// the same for cc capture channels and int16 (s16) or float samples
KernelRef v3_kernel(int N, int cc, int R, int extra, bool s16, const KParams &kp, bool display);
} // namespace wf
