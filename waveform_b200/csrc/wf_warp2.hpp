// wf_warp2.hpp — host interface of the warp-per-stream kernel for fft sizes N = 2*L*P (wf_warp2.cuh)
#pragma once
#include <cstddef>

namespace wf {

// The compiled (L, P) plan of one fft size.  L == 0: the size has none.  Its kernels launch with programmatic dependent
// launch, 32 threads per warp.
struct Warp2Plan {
    int L = 0, P = 0;
    int table_bytes = 0, warp_bytes = 0;   // shared memory per CTA and per warp of the plain kernel
    const void *kernel[2][2][2] = {};      // stft_warp2_kernel<L, P, extra, disp, TS>, [s16][extra][disp]: s16 = int16 samples
                                           // (wf_pcm.cuh); extra = slope / fast peaks / skip mask / volume / roll-off / peak
                                           // output in use; disp = display outputs (points / pixels / minimum) requested

    // a CTA of `warps` warps, with the display variant's per-CTA tables and per-warp rows (0 for the plain kernel)
    size_t smem_bytes(int warps, size_t disp_tab_bytes, size_t disp_warp_bytes) const
    {
        return (size_t)table_bytes + disp_tab_bytes + (size_t)warps * (warp_bytes + disp_warp_bytes);
    }
};

// The plan for this fft size: the non-power-of-two sizes, and 512 / 1024 / 2048 (routed here only for display outputs)
Warp2Plan warp2_plan(int N);
} // namespace wf
