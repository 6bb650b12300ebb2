// wf_fast2048.hpp — host interface of the N=2048 warp-per-stream kernel (wf_fast2048.cuh): its shared-memory layout, which
// routing and the launch size CTAs by, and the lookup of its instantiations (wf_fast2048.cu)
#pragma once
#include "wf_host.hpp"

namespace wf {

namespace fast {

constexpr int kN = 2048;
constexpr int kM = 1024;
// Per warp, in this order: the TMA landing buffer of the next frame (8 KiB); the padded transpose buffer, which after
// pass B stages the frame's dB row for its bulk store (8448 B); the mbarrier and the split-mode hand-over flag (16 B).
// Every part is 16-byte aligned.  The EMA state of the stream lives in registers.
constexpr int kLandBytes = kN * 4;
constexpr int kXposeBytes = 32 * 33 * 8;
constexpr int kWarpBytes = kLandBytes + kXposeBytes + 16;
constexpr int kTableBytes = (1024 + 1024 + 512) * 8;
constexpr int kMaxWarpsPerCta = 12; // 1 CTA/SM: 12 warps x 16.3 KB + 20 KB tables = 215 KB of shared memory, 168 registers/thread
constexpr int smem_bytes(int warps_per_cta) { return kTableBytes + warps_per_cta * kWarpBytes; }
static_assert(smem_bytes(kMaxWarpsPerCta) <= 227 * 1024, "one CTA per SM must fit");

} // namespace fast

// stft2048_fast_kernel<kMaxWarpsPerCta, tsm, gate, extra, int16 (s16) or float samples>, with the CTA size and shared memory
// of kMaxWarpsPerCta warps.  tsm = temporal smoothing, gate = silence gate, extra = slope / fast peaks / skip mask / volume /
// roll-off / peak output in use.  A launch of w <= kMaxWarpsPerCta warps per CTA takes w * 32 threads and smem_bytes(w).  It
// launches with programmatic dependent launch, at most one CTA per SM.
KernelRef fast2048_kernel(bool tsm, bool gate, bool extra, bool s16);

} // namespace wf
