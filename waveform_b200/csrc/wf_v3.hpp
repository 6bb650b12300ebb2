// wf_v3.hpp — host interface of the CTA-per-tick kernel for fft sizes 4096 / 8192 / 16384 (wf_v3.cuh)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <vector>

namespace wf {
struct KParams;
bool v3_supported(int N);
int v3_min_cluster(int N); // smallest supported cluster size (1, or 2 where the per-thread state would not fit registers)
size_t v3_smem_bytes(int N, int dch, int n_points, bool display, int cc, int R);
// Inter-pass twiddle tables (interleaved re,im), evaluated in double: tw1[ka][t] = W_M^(t*ka), tw2[kb][c] = W_(BC)^(c*kb);
// tw0 (16384 only) = W_M^(a*TN + t) of the radix-2 first stage, tw1/tw2 then belong to the 4096-point sub-FFTs
void v3_build_twiddles(int N, std::vector<float> &tw1, std::vector<float> &tw2, std::vector<float> &tw0);
// R = CTAs per stream (1 = no cluster); extra: 0 = plain, 1 = per-tick peak output only, 3 = slope / fast peaks / skip mask /
// volume / roll-off in use (with or without the peak output); s16 = int16 samples
cudaError_t v3_launch(int N, int cc, int R, int extra, bool s16, const KParams &kp, const float *d_tw1, const float *d_tw2,
                      const float *d_tw0, cudaStream_t st, bool display, int device);
} // namespace wf
