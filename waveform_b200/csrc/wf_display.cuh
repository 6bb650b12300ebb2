// wf_display.cuh — the dB -> pixel step shared by the waveform and level-meter display stages (render_curve / render_bars,
// src/source.cpp:1410, :1550):  val = lerp(top, bottom, clamp(ceiling - db, 0, range) / range), no contraction.
// The spectrum path does the same inline in display_stage_tab (wf_kernels.cuh).
#pragma once
#include <cuda_runtime.h>

#include "wf_kernels.cuh" // std_lerp_dev: std::lerp as libstdc++ evaluates it

namespace wf {

// pixel height of one dB value: std::clamp(ceiling - db, 0, range) / range, then the lerp
__device__ __forceinline__ float display_pixel(float db, float ceiling, float range, float top, float bottom)
{
    const float x = __fsub_rn(ceiling, db);
    const float c = (x < 0.0f) ? 0.0f : ((range < x) ? range : x);
    return std_lerp_dev(top, bottom, __fdiv_rn(c, range));
}

} // namespace wf
