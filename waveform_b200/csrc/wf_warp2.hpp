// wf_warp2.hpp — host interface of the warp-per-stream kernel for fft sizes N = 2*L*P (wf_warp2.cuh)
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace wf {
struct KParams;

// grid = CTAs, warps = warps per CTA, smem = dynamic shared memory bytes (smem_bytes below)
using Warp2Launch = cudaError_t (*)(const KParams &kp, int grid, int warps, size_t smem, cudaStream_t st, int device);

// The compiled (L, P) plan of one fft size.  L == 0: the size has none.
struct Warp2Plan {
    int L = 0, P = 0;
    int table_bytes = 0, warp_bytes = 0; // shared memory per CTA and per warp of the plain kernel
    Warp2Launch launch[2][2][2] = {};    // [s16][extra][disp]: s16 = int16 samples (wf_pcm.cuh); extra = slope / fast peaks /
                                         // skip mask / volume / roll-off / peak output in use; disp = display outputs (points /
                                         // pixels / minimum) requested

    // a CTA of `warps` warps, with the display variant's per-CTA tables and per-warp rows (0 for the plain kernel)
    size_t smem_bytes(int warps, size_t disp_tab_bytes, size_t disp_warp_bytes) const
    {
        return (size_t)table_bytes + disp_tab_bytes + (size_t)warps * (warp_bytes + disp_warp_bytes);
    }
};

// The plan for this fft size: the non-power-of-two sizes, and 512 / 1024 / 2048 (routed here only for display outputs)
Warp2Plan warp2_plan(int N);
} // namespace wf
