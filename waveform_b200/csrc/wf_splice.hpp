// wf_splice.hpp — the per-stream history all three engines keep between calls: the spectrum engine's capture ring
// (wf_batch.capture_ring), the level meter's sync-offset delay line and the waveform's sync-offset holdback.
//
// Each (stream, capture channel) has a history of R float samples, oldest first.  A call brings L new samples per channel, and
// the engine's kernels read a window of the timeline  C = history ++ new  (length R + L):
//   window := C[ws .. ws + wl)   in the call's sample type (an int16 call sees the float history rounded to int16)
//   history := C[L .. L + R)     the last R samples of C
// The engine's own kernels then run unchanged on the window as if it were the caller's PCM.
#pragma once
#include <cuda_runtime.h>

#include <stdint.h>

#include "wf_host.hpp"
#include "wfstft.h"

namespace wf {

struct Splice {
    float *hist;                             // [streams][cc][R]
    void *win;                               // [streams][cc][win_cs] in the call's sample type; null: no window, and then
                                             // L >= R (the history is all new samples; the kernels read those in place)
    const void *pcm;                         // the call's new samples, in its sample type
    long long stream_stride, channel_stride; // of pcm, in samples
    long long win_cs;                        // samples per (stream, channel) of win
    long long ws, wl;                        // the window; with win: ws <= L and ws + wl >= R (the history the next call
                                             // keeps and that predates the call lies in the window)
    long long L;                             // new samples per (stream, channel)
    int R;                                   // history length (>= 1)
    // A spectrum ring call whose slots may still owe samples to the sync offset (else owed is null): the call's skip_mask
    // is written here from the device-side counts, which then drop by L, so that a replayed graph skips each slot's start-up
    // ticks exactly once, as the same sequence of eager calls does.
    long long *owed;                         // [streams] samples each slot still needs before its first real tick
    unsigned char *mask;                     // [streams][T] := (t < start-up ticks of the slot) | caller[s][t]
    const unsigned char *caller;             // [streams][T] the caller's skip_mask, or null
    int T, hop;                              // ticks of the call, samples between ticks
};

// One CTA per (stream, channel) of `streams` x `cc`, on stream `st` of `device`.  Returns the launch's error.
cudaError_t launch_splice(const Splice &s, int device, int streams, int cc, bool s16, cudaStream_t st);

// The window stride of `len` samples: rounded up to 16 bytes, so that a window keeps 16-byte alignment wherever the
// kernels' own facts (hop, strides) allow it.
inline long long splice_stride(long long len, bool s16)
{
    const long long q = s16 ? 8 : 4;
    return (len + q - 1) / q * q;
}

// The sync-offset holdback of the level meter and the waveform: the splice with ws = 0 and no start-up mask, for `streams`
// x `cc` rows of `view` with L new samples each.  `hist` holds R samples per row from the call's first stream on; `window`
// grows to the call's window of wl samples per row.  Counts the launch, then points `view` at the window, which the
// engine's kernels read instead of the call's PCM.
int splice_holdback(HostCore *c, float *hist, int R, int streams, int cc, long long L, long long wl, bool s16,
                    DevBuf<float> &window, PcmView &view, cudaStream_t st);

// The samples an audio sync offset of `ms` milliseconds holds back: ns_to_audio_frames(sample_rate, ms * 10^6) for a
// positive offset (get_audio_sync > 0), else 0.
inline int sync_delay(uint32_t sample_rate, int32_t ms)
{
    return ms > 0 ? (int)(((unsigned __int128)((uint64_t)ms * 1000000ull) * sample_rate) / 1000000000ull) : 0;
}

// The plugin's slider range (src/source.cpp:195), which also bounds the engines' delay memory.
inline bool sync_offset_ok(int32_t ms) { return ms >= -1000 && ms <= 1000; }

} // namespace wf
