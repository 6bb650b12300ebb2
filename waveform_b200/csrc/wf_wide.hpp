// wf_wide.hpp — host interface of the cluster kernel (wf_wide.cuh / wf_wide.cu)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace wf {
struct KParams;
bool wide_supported(int N);
size_t wide_smem_bytes(int N, int dch, int n_points, bool display);
// R = cluster size (2, 4 or 8 CTAs per stream); grid = n_streams * R; s16 = int16 samples
cudaError_t wide_launch(int N, int cc, int R, bool s16, const KParams &kp, cudaStream_t st, bool display, int device);
} // namespace wf
