// wf_wave.cu — waveform (oscilloscope) mode of the plugin (tick_waveform) as a batched sm_90a gather behind the C ABI of
// include/wfstft.h (wf_wave_*).  SURVEY.md §8(f) rank 4.
//
// Reference semantics restated (paths relative to the reference tree): src/source_generic.cpp:272-390 with the capture side
// of src/source.cpp:1817-1888 for packets that end "now"; setup src/source.cpp:1129-1143, :1181, :1243-1248.
//
// The reference walks a nanosecond clock: every tick it emits the points whose timestamps m_waveform_ts + i*step_ns fall
// into the span of the audio captured since the last tick and picks the NEAREST sample for each.  All of that arithmetic is
// independent of the audio itself, so the host plans a call once (plan_ticks: per tick the number of new points and, for
// each, which sample of the packet it takes — integer arithmetic, bit-exact; on an engine created with device_clock = 1,
// wave_plan_kernel makes the same plan on the device) and the device does what is left per stream:
// gather the samples, keep the scrolling buffer (a ring in shared memory), evaluate the all-zero "silent" rule, convert
// the new points to dBFS (|x|, stereo / mono mix), add the volume compensation, and write the buffer row of every tick.
// HBM traffic: the packet's sectors once in, width floats per display channel and tick out.  The kernels take the sample
// type of the PCM (float or int16_t, wf_wave_batch.pcm_format) as their last template argument and gather it only through
// Pcm<TS> (wf_pcm.cuh); everything after the gather (buffers, silent rule, dBFS, display) sees the widened floats, so an
// int16 call and the float call on the same values agree bit for bit.  There is no CPU fallback.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "wf_display.cuh"
#include "wf_host.hpp"
#include "wf_splice.hpp"
#include "wf_nvtx.hpp"
#include "wf_pcm.cuh"
#include "wf_tables.hpp"
#include "wfstft.h"

namespace {

struct WParams {
    const float *pcm;
    long long stream_stride, channel_stride;
    const float *input_rms;  // [streams][ticks] or null
    const int *src;          // flat: for tick t, points [off[t], off[t+1]): sample index into the call's PCM, or -1 = start-up zero
    const int *off;          // [ticks + 1]
    float *state;            // [streams][2][width] scrolling buffers, oldest point first
    unsigned char *flags;    // [streams] m_last_silent
    float *out;              // [streams][ticks][dch][width]
    unsigned char *out_silent;
    int n_streams, n_ticks, width, cc, dch, och, stereo, normalize;
    float vol_target, max_gain, db_min;
};
// The parameters of the kernels with the display stage (the plain kernels keep WParams, and with it their code):
// tables of wf::build_wave_tables, the display outputs, render_curve's geometry.
struct WDisp : WParams {
    const float *interp_w;    // [width][taps] or null (point mode); 16-byte aligned
    const float *interp_idx;  // [width]
    const float *gauss_w;     // [2 * gauss_radius - 1] or null
    float *out_points;        // [streams][ticks][dch][width] or null
    float *out_pixels;        // same shape or null
    float *out_min;           // [streams][ticks][2] or null
    int taps, filter, gauss_radius, scratch_off; // scratch_off: floats of dynamic shared memory before the Gaussian's scratch row
    int vec4;                 // width % 4 == 0 and 16-byte aligned display outputs: float4 stores
    float gauss_sum, ceiling_f, dbrange_f, px_hi, px_cpos;
};

__device__ __forceinline__ float dbfs_dev(float mag, float db_min) { return (mag > 0.0f) ? 20.0f * log10f(mag) : db_min; }

// ---- display stage: render_curve in waveform mode (src/source.cpp:1375-1417) for the rows of one or more ticks ---------------
// The operation order is the spectrum path's display_stage_tab / kernel_sum / weighted_avg (wf_kernels.cuh), which are pinned
// against the reference; restated here because a waveform row is a window of a ring in shared memory, not a contiguous array.

// One display row: element k is a[(a0 + k) mod cap] for k < split and b[k] from there on (the one-channel-shown-as-two layout's
// second row: older points from the dB ring, the tick's own points raw); a silent row is DB_MIN throughout.  Built once per
// (tick, channel, point group), so the taps only add k.
struct RowSeg {
    const float *a, *b;
    int a0, cap, split;
    bool sil;
    float fill;
    __device__ __forceinline__ float operator()(int k) const
    {
        if(sil)
            return fill;
        if(k < split)
        {
            const int x = a0 + k;
            return a[x - ((x >= cap) ? cap : 0)];
        }
        return b[k];
    }
};

// interpolated dB of display point i.  TAPS 0: point mode, the sample at (int)m_interp_indices[i] (:1393-1394; std::lerp puts
// some indices just below an integer, so that is sample i - 1 there).  TAPS 4 / 8: Catmull-Rom / Lanczos, kernel_convolve
// (src/filter.hpp:160-169): taps outside [0, width) are skipped, the rest summed in tap order; the weights come in 128-bit loads
// (the table is 16-byte aligned and a point has 4 or 8 of them).
template<int TAPS>
__device__ __forceinline__ float wave_interp(const WDisp &p, const RowSeg &row, int i)
{
    const int index = (int)__ldg(p.interp_idx + i);
    if constexpr(TAPS == 0)
        return row(index);
    else
    {
        float wt[TAPS];
        const float4 *w4 = reinterpret_cast<const float4 *>(p.interp_w) + (size_t)i * (TAPS / 4);
#pragma unroll
        for(int q = 0; q < TAPS / 4; ++q)
        {
            const float4 v = __ldg(w4 + q);
            wt[4 * q] = v.x;
            wt[4 * q + 1] = v.y;
            wt[4 * q + 2] = v.z;
            wt[4 * q + 3] = v.w;
        }
        const int start = index - TAPS / 2 + 1;
        float sum = 0.0f;
#pragma unroll
        for(int k = 0; k < TAPS; ++k)
        {
            const int j = start + k;
            if((unsigned)j < (unsigned)p.width)
                sum = __fadd_rn(sum, __fmul_rn(row(j), wt[k]));
        }
        return sum;
    }
}

// weighted_avg (src/filter.hpp:133-158): the Gaussian, renormalised where it overhangs the row's ends
__device__ __forceinline__ float wave_gauss(const WDisp &p, const float *raw, int i)
{
    const int n = p.width, start = (i - p.gauss_radius) + 1, stop = i + p.gauss_radius;
    float sum = 0.0f;
    if((start < 0) || (stop > n))
    {
        float wsum = 0.0f;
        for(int k = max(start, 0); k < min(stop, n); ++k)
        {
            const float weight = __ldg(p.gauss_w + (k - start));
            wsum = __fadd_rn(wsum, weight);
            sum = __fadd_rn(sum, __fmul_rn(raw[k], weight));
        }
        return __fdiv_rn(sum, wsum);
    }
    for(int k = start; k < stop; ++k)
        sum = __fadd_rn(sum, __fmul_rn(raw[k], __ldg(p.gauss_w + (k - start))));
    return __fdiv_rn(sum, p.gauss_sum);
}

// stores points [i, i + V) of display channel d of tick t (one float4 per output when V = 4) and returns their arg-min key:
// pixel heights are >= +0, so the float's bits order like the value, and the low word (channel, index) makes ties go to the
// earliest point, as the sequential scan does
template<int V>
__device__ __forceinline__ unsigned long long wave_emit(const WDisp &p, int s, int t, int d, int i, const float (&db)[V])
{
    const size_t o = (((size_t)s * p.n_ticks + t) * p.dch + d) * p.width + i;
    float px[V];
    unsigned long long key = ~0ull;
#pragma unroll
    for(int u = 0; u < V; ++u)
    {
        px[u] = wf::display_pixel(db[u], p.ceiling_f, p.dbrange_f, 0.0f, p.px_hi);
        key = min(key, ((unsigned long long)__float_as_uint(px[u]) << 32) | (unsigned)(d * p.width + i + u));
    }
    if constexpr(V == 4)
    {
        if(p.out_points != nullptr)
            __stcs(reinterpret_cast<float4 *>(p.out_points + o), make_float4(db[0], db[1], db[2], db[3]));
        if(p.out_pixels != nullptr)
            __stcs(reinterpret_cast<float4 *>(p.out_pixels + o), make_float4(px[0], px[1], px[2], px[3]));
    }
    else
    {
        if(p.out_points != nullptr)
            __stcs(p.out_points + o, db[0]);
        if(p.out_pixels != nullptr)
            __stcs(p.out_pixels + o, px[0]);
    }
    return key;
}

// Without the Gaussian: every (tick, channel, group of V points) of ticks [t0, t0 + K) at once.  A thread's items come in tick
// order (the item index walks by nt; no division per item), so it folds its keys per tick before the shared atomic.
template<int TAPS, int V, class Seg>
__device__ __forceinline__ void wave_display_points(const WDisp &p, const Seg &seg, int s, int t0, int K,
                                                    unsigned long long *s_min, int tid, int nt)
{
    const int Wv = p.width / V, per = p.dch * Wv;
    int j = tid / per, r = tid - j * per, jc = -1;
    unsigned long long key = ~0ull;
    while(j < K)
    {
        const int d = (r >= Wv) ? 1 : 0, i = (r - d * Wv) * V;
        if(j != jc)
        {
            if(jc >= 0)
                atomicMin(&s_min[jc], key);
            jc = j;
            key = ~0ull;
        }
        const RowSeg row = seg(j, d);
        float v[V];
#pragma unroll
        for(int u = 0; u < V; ++u)
            v[u] = wave_interp<TAPS>(p, row, i + u);
        key = min(key, wave_emit<V>(p, s, t0 + j, d, i, v));
        r += nt;
        while(r >= per)
        {
            r -= per;
            ++j;
        }
    }
    if(jc >= 0)
        atomicMin(&s_min[jc], key);
}

// With the Gaussian: one tick at a time through the scratch row(s) (the Gaussian reads its neighbours' interpolated values).
template<int TAPS, class Seg>
__device__ __forceinline__ void wave_display_gauss(const WDisp &p, const Seg &seg, int s, int t0, int K, float *scratch,
                                                   unsigned long long *s_min, int tid, int nt)
{
    const int W = p.width, per = p.dch * W;
    for(int j = 0; j < K; ++j)
    {
        __syncthreads(); // the previous tick's scratch reads are done
        for(int r = tid; r < per; r += nt)
        {
            const int d = (r >= W) ? 1 : 0;
            scratch[r] = wave_interp<TAPS>(p, seg(j, d), r - d * W);
        }
        __syncthreads();
        unsigned long long key = ~0ull;
        for(int r = tid; r < per; r += nt)
        {
            const int d = (r >= W) ? 1 : 0, i = r - d * W;
            const float v[1] = {wave_gauss(p, scratch + d * W, i)};
            key = min(key, wave_emit<1>(p, s, t0 + j, d, i, v));
        }
        if(key != ~0ull)
            atomicMin(&s_min[j], key);
    }
}

// The display stage of ticks [t0, t0 + K) of stream s, K <= WCH_KMAX; seg(j, d) is the RowSeg of display channel d of tick
// t0 + j.  Called by all threads of the CTA; s_min: K keys of shared memory; scratch: dch * width floats (Gaussian only).
template<class Seg>
__device__ __forceinline__ void wave_display(const WDisp &p, const Seg &seg, int s, int t0, int K, float *scratch,
                                             unsigned long long *s_min, int tid, int nt)
{
    if(tid < K)
        s_min[tid] = ~0ull;
    __syncthreads();
    if(p.filter)
    {
        if(p.taps == 0)
            wave_display_gauss<0>(p, seg, s, t0, K, scratch, s_min, tid, nt);
        else if(p.taps == 4)
            wave_display_gauss<4>(p, seg, s, t0, K, scratch, s_min, tid, nt);
        else
            wave_display_gauss<8>(p, seg, s, t0, K, scratch, s_min, tid, nt);
    }
    else if(p.vec4)
    {
        if(p.taps == 0)
            wave_display_points<0, 4>(p, seg, s, t0, K, s_min, tid, nt);
        else if(p.taps == 4)
            wave_display_points<4, 4>(p, seg, s, t0, K, s_min, tid, nt);
        else
            wave_display_points<8, 4>(p, seg, s, t0, K, s_min, tid, nt);
    }
    else
    {
        if(p.taps == 0)
            wave_display_points<0, 1>(p, seg, s, t0, K, s_min, tid, nt);
        else if(p.taps == 4)
            wave_display_points<4, 1>(p, seg, s, t0, K, s_min, tid, nt);
        else
            wave_display_points<8, 1>(p, seg, s, t0, K, s_min, tid, nt);
    }
    __syncthreads();
    if(p.out_min != nullptr && tid < K)
    {
        // miny starts at cpos and only a strictly smaller value replaces it; minpos is the index within its channel
        const unsigned long long key = s_min[tid];
        const float v = __uint_as_float((unsigned)(key >> 32));
        const bool lt = v < p.px_cpos;
        float *o = p.out_min + ((size_t)s * p.n_ticks + t0 + tid) * 2;
        o[0] = lt ? v : p.px_cpos;
        o[1] = lt ? (float)((int)(key & 0xffffffffu) % p.width) : 0.0f;
    }
}

// One CTA per stream; the scrolling buffers live in shared memory as rings (head = oldest point).  DISP: with the display
// stage after every tick (out may then be null).
template<class P, typename TS>
__global__ void __launch_bounds__(256, std::is_same_v<P, WDisp> ? 4 : 0) wave_kernel(const P p)
{
    constexpr bool DISP = std::is_same_v<P, WDisp>;
    extern __shared__ float ring[]; // [2][width] (DISP with the Gaussian: then the scratch row(s))
    const int W = p.width, tid = threadIdx.x, nt = blockDim.x;
    for(int s = blockIdx.x; s < p.n_streams; s += gridDim.x)
    {
        float *r0 = ring, *r1 = ring + W;
        for(int i = tid; i < 2 * W; i += nt)
            ring[i] = p.state[(size_t)s * 2 * W + i];
        int head = 0;
        bool last_silent = p.flags[s] != 0;
        const TS *pcm0 = wf::Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride;
        const TS *pcm1 = pcm0 + p.channel_stride;
        __syncthreads();
        for(int t = 0; t < p.n_ticks; ++t)
        {
            const int o0 = p.off[t], cnt = p.off[t + 1] - o0;
            // the cnt oldest points are replaced by the new raw samples, then the ring rotates (src/source_generic.cpp:333-339)
            for(int i = tid; i < cnt; i += nt)
            {
                const int q = __ldg(p.src + o0 + i);
                int pos = head + i;
                pos -= (pos >= W) ? W : 0;
                r0[pos] = (q >= 0) ? wf::Pcm<TS>::ldg1(pcm0 + q) : 0.0f;
                if(p.cc > 1)
                    r1[pos] = (q >= 0) ? wf::Pcm<TS>::ldg1(pcm1 + q) : 0.0f;
            }
            head += cnt;
            head -= (head >= W) ? W : 0;
            __syncthreads();
            // "silent" = every entry of the channel's buffer is exactly 0.0f (:341-356)
            bool nz0 = false, nz1 = false;
            for(int i = tid; i < W; i += nt)
            {
                nz0 |= (r0[i] != 0.0f);
                if(p.cc > 1)
                    nz1 |= (r1[i] != 0.0f);
            }
            const bool any0 = __syncthreads_or(nz0 ? 1 : 0) != 0;
            const bool any1 = (p.cc > 1) ? (__syncthreads_or(nz1 ? 1 : 0) != 0) : false;
            unsigned silent_channels = 0;
            if(any0)
                last_silent = false;
            else if(++silent_channels >= (unsigned)p.cc)
                last_silent = true;
            if(p.cc > 1)
            {
                if(any1)
                    last_silent = false;
                else if(++silent_channels >= (unsigned)p.cc)
                    last_silent = true;
            }
            if(last_silent)
            {
                for(int i = tid; i < p.dch * W; i += nt)
                    ring[i] = p.db_min; // :360-366 (display channels only)
            }
            else
            {
                if(p.och > p.cc) // mono capture shown as two channels: whole-buffer copy (:368-369)
                    for(int i = tid; i < W; i += nt)
                        r1[i] = r0[i];
                __syncthreads();
                float vc = 0.0f;
                if(p.normalize)
                {
                    const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * p.n_ticks + t] : 0.0f;
                    vc = fminf(p.vol_target - dbfs_dev(rms, p.db_min), p.max_gain);
                }
                // the new points are the last cnt of the rotated buffer (:371-388)
                for(int i = tid; i < cnt; i += nt)
                {
                    int pos = head - cnt + i;
                    pos += (pos < 0) ? W : 0;
                    if(p.stereo)
                    {
                        float a = dbfs_dev(fabsf(r0[pos]), p.db_min);
                        if(p.normalize)
                            a += vc;
                        r0[pos] = a;
                        // counts[1] stays 0 for a single capture channel (:371-375): the second display channel keeps
                        // the RAW new samples of the whole-buffer copy above — reproduced as is
                        if(p.cc > 1)
                        {
                            float b = dbfs_dev(fabsf(r1[pos]), p.db_min);
                            if(p.normalize)
                                b += vc;
                            r1[pos] = b;
                        }
                    }
                    else
                    {
                        float a = (p.cc > 1) ? dbfs_dev((fabsf(r0[pos]) + fabsf(r1[pos])) * 0.5f, p.db_min)
                                             : dbfs_dev(fabsf(r0[pos]), p.db_min);
                        if(p.normalize)
                            a += vc;
                        r0[pos] = a;
                    }
                }
            }
            __syncthreads();
            // the tick's row(s): buffer in time order
            if(!DISP || p.out != nullptr)
            {
                float *orow = p.out + ((size_t)s * p.n_ticks + t) * p.dch * W;
                for(int d = 0; d < p.dch; ++d)
                    for(int i = tid; i < W; i += nt)
                    {
                        int pos = head + i;
                        pos -= (pos >= W) ? W : 0;
                        __stcs(orow + d * W + i, ring[d * W + pos]);
                    }
            }
            if(p.out_silent != nullptr && tid == 0)
                p.out_silent[(size_t)s * p.n_ticks + t] = last_silent ? 1 : 0;
            if constexpr(DISP)
            {
                __shared__ unsigned long long s_min[1];
                const int hd = head;
                wave_display(
                    p, [&](int, int d) { return RowSeg{ring + d * W, ring, hd, W, W, false, 0.0f}; }, s, t, 1,
                    ring + p.scratch_off, s_min, tid, nt);
            }
            __syncthreads();
        }
        for(int i = tid; i < 2 * W; i += nt)
        {
            int pos = head + (i % W);
            pos -= (pos >= W) ? W : 0;
            p.state[(size_t)s * 2 * W + i] = ring[(i / W) * W + pos];
        }
        if(tid == 0)
            p.flags[s] = last_silent ? 1 : 0;
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Chunked form of the same tick loop.  The per-tick kernel above has ~90 gathers in flight per CTA between barriers, so it
// is latency-bound; here a CTA takes as many consecutive ticks as bring in at most `width` new points, gathers and converts
// ALL of them at once (warp per 32 points, every load of the chunk in flight together), and writes each tick's row as a
// sliding window over the extended buffer  E = [scrolling buffer at chunk start | new points of the chunk]  kept as a ring of
// 2*width floats per channel.  The all-zero "silent" rule needs, per tick, whether the window holds any non-zero entry:
// that is a running count  (window count) - (non-zeros leaving with this tick) + (non-zeros entering), and the per-tick
// leaving / entering counts are accumulated by the gather warps with ballots.  A tick that does turn silent ends the chunk
// early (the buffer becomes DB_MIN and the following ticks must see that); that is the rare path.
//   MODE 0: one capture channel, one display channel           E0
//   MODE 1: two capture channels mixed to one display channel  E0 (dB of the mix), E1 (RAW second channel: the reference's
//           mono branch never converts m_decibels[1], src/source_generic.cpp:380-388 — it only takes part in the silent rule)
//   MODE 2: two capture channels, two display channels         E0, E1 (both dB)
//   MODE 3: one capture channel shown as two                   E0 and the raw new points N0: row 1 of a tick is the whole-buffer
//           copy taken BEFORE the tick's conversion (:368-369), i.e. older points in dB, the tick's own points raw
constexpr int WCH_KMAX = 32; // ticks per chunk: one lane each in the gather phase
constexpr int WCH_U = 4;     // items (32 points) a warp has in flight

struct WChunkTick {
    int leave0, in_db0, in_raw0, leave1, in1, in_raw1;
};

__device__ __forceinline__ int wrap2(int x, int cap) { return x - ((x >= cap) ? cap : 0); }

// DISP: the display stage runs over the rows of every chunk after they are stored (out may then be null).  Its instantiations
// get 64 registers (4 CTAs per SM) instead of 48: the plain ones keep their budget.
template<int MODE, class P, typename TS>
__global__ void __launch_bounds__(256, std::is_same_v<P, WDisp> ? 4 : 5) wave_chunk_kernel(const P p)
{
    constexpr bool DISP = std::is_same_v<P, WDisp>;
    extern __shared__ float wsm[];
    __shared__ WChunkTick s_cnt[2][WCH_KMAX];
    __shared__ int s_off[WCH_KMAX + 1];
    constexpr bool TWO = (MODE == 1 || MODE == 2); // second capture channel present
    constexpr int DCH = (MODE >= 2) ? 2 : 1;
    constexpr int nt = 256, nwarps = nt / 32; // the launch uses exactly 256 threads
    const int W = p.width, CAP = 2 * W, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    float *E0 = wsm;
    float *E1 = wsm + CAP;                               // MODE 1, 2
    float *N0 = wsm + CAP;                               // MODE 3 (raw new points of the chunk, chunk-relative index)
    const bool vec = ((W & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0);
    for(int s = blockIdx.x; s < p.n_streams; s += gridDim.x)
    {
        const TS *pcm0 = wf::Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride;
        const TS *pcm1 = pcm0 + p.channel_stride;
        float *st0 = p.state + (size_t)s * 2 * W, *st1 = st0 + W;
        int wc0 = 0, wc1 = 0; // non-zero entries in the current window of E0 / E1
        {
            int c0 = 0, c1 = 0;
            for(int i = tid; i < W; i += nt)
            {
                const float a = st0[i];
                E0[i] = a;
                c0 += (a != 0.0f);
                if(TWO)
                {
                    const float b = st1[i];
                    E1[i] = b;
                    c1 += (b != 0.0f);
                }
            }
            if(tid < 2 * WCH_KMAX)
                reinterpret_cast<WChunkTick *>(s_cnt)[tid] = WChunkTick{0, 0, 0, 0, 0, 0};
            // block sums (once per stream and call)
            for(int o = 16; o > 0; o >>= 1)
            {
                c0 += __shfl_xor_sync(0xffffffffu, c0, o);
                c1 += __shfl_xor_sync(0xffffffffu, c1, o);
            }
            __shared__ int s_red[2][8];
            if(lane == 0)
            {
                s_red[0][warp] = c0;
                s_red[1][warp] = c1;
            }
            __syncthreads();
            for(int w = 0; w < nwarps; ++w)
            {
                wc0 += s_red[0][w];
                wc1 += s_red[1][w];
            }
        }
        int base = 0, par = 0;
        bool last_silent = p.flags[s] != 0;
        int t = 0;
        while(t < p.n_ticks)
        {
            // the chunk: ticks [t, t+K) with at most W new points in total (the first tick is always taken: a tick never
            // brings more than W points)
            // (lane l looks at tick t+l: the cumulative point counts are monotone, so the chunk is a ballot)
            const int obase = __ldg(p.off + t);
            const bool tick_l = (t + lane) < p.n_ticks;
            const int cum_l = tick_l ? (__ldg(p.off + t + lane + 1) - obase) : 0x3fffffff;
            const int K = max(1, __popc(__ballot_sync(0xffffffffu, tick_l && cum_l <= W)));
            const int C = __shfl_sync(0xffffffffu, cum_l, K - 1);
            // phase 1: gather + convert, one warp per item of 32 points, WCH_U items per pass so that a warp has that many
            // dependent src -> sample load chains in flight; per-tick leaving / entering non-zero counts by ballot.
            // Lane l holds tick l's offsets; an item number maps to its tick through a ballot over the running item ends.
            {
                int oj_l = __shfl_up_sync(0xffffffffu, cum_l, 1), c_l = 0;
                if(lane == 0)
                    oj_l = 0;
                if(lane < K)
                    c_l = cum_l - oj_l;
                else
                    oj_l = 0;
                const int nb_l = (c_l + 31) >> 5;
                int end_l = nb_l;
#pragma unroll
                for(int o = 1; o < 32; o <<= 1)
                {
                    const int v = __shfl_up_sync(0xffffffffu, end_l, o);
                    end_l += (lane >= o) ? v : 0;
                }
                const int total = __shfl_sync(0xffffffffu, end_l, 31);
                if(warp == 0)
                {
                    if(lane < K)
                        s_off[lane + 1] = oj_l + c_l;
                    if(lane == 0)
                        s_off[0] = 0;
                    s_cnt[par ^ 1][lane] = WChunkTick{0, 0, 0, 0, 0, 0}; // the next chunk's counters (last read two barriers ago)
                }
                for(int g0 = warp; g0 < total; g0 += nwarps * WCH_U)
                {
                    int jj[WCH_U], rel[WCH_U], q[WCH_U];
                    float ra[WCH_U], rb[WCH_U];
#pragma unroll
                    for(int u = 0; u < WCH_U; ++u)
                    {
                        const int g = g0 + u * nwarps;
                        const int j = min(__popc(__ballot_sync(0xffffffffu, lane < K && end_l <= g)), K - 1);
                        const int oj = __shfl_sync(0xffffffffu, oj_l, j), c = __shfl_sync(0xffffffffu, c_l, j);
                        const int first = __shfl_sync(0xffffffffu, end_l - nb_l, j);
                        const int i = (g - first) * 32 + lane;
                        const bool act = (g < total) && (i < c);
                        jj[u] = (g < total) ? j : -1;
                        rel[u] = act ? (oj + i) : -1;
                        q[u] = act ? __ldg(p.src + obase + oj + i) : -1;
                    }
#pragma unroll
                    for(int u = 0; u < WCH_U; ++u)
                    {
                        ra[u] = (q[u] >= 0) ? wf::Pcm<TS>::ldg1(pcm0 + q[u]) : 0.0f;
                        rb[u] = (TWO && q[u] >= 0) ? wf::Pcm<TS>::ldg1(pcm1 + q[u]) : 0.0f;
                    }
#pragma unroll
                    for(int u = 0; u < WCH_U; ++u)
                    {
                        if(jj[u] < 0)
                            continue; // warp-uniform
                        const bool act = rel[u] >= 0;
                        float vc = 0.0f;
                        if(p.normalize)
                        {
                            const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * p.n_ticks + t + jj[u]] : 0.0f;
                            vc = fminf(p.vol_target - dbfs_dev(rms, p.db_min), p.max_gain);
                        }
                        const int pl = wrap2(base + max(rel[u], 0), CAP), pn = wrap2(base + W + max(rel[u], 0), CAP);
                        const bool l0 = act && (E0[pl] != 0.0f);
                        const bool l1 = TWO && act && (E1[pl] != 0.0f);
                        float a, b1 = 0.0f;
                        if(MODE == 1)
                            a = dbfs_dev((fabsf(ra[u]) + fabsf(rb[u])) * 0.5f, p.db_min);
                        else
                            a = dbfs_dev(fabsf(ra[u]), p.db_min);
                        if(p.normalize)
                            a += vc;
                        if(MODE == 2)
                        {
                            b1 = dbfs_dev(fabsf(rb[u]), p.db_min);
                            if(p.normalize)
                                b1 += vc;
                        }
                        else if(MODE == 1)
                            b1 = rb[u];
                        if(act)
                        {
                            E0[pn] = a;
                            if(TWO)
                                E1[pn] = b1;
                            if(MODE == 3)
                                N0[rel[u]] = ra[u];
                        }
                        const unsigned m_l0 = __ballot_sync(0xffffffffu, l0), m_a = __ballot_sync(0xffffffffu, act && a != 0.0f),
                                       m_ra = __ballot_sync(0xffffffffu, act && ra[u] != 0.0f);
                        unsigned m_l1 = 0, m_b = 0, m_rb = 0;
                        if(TWO)
                        {
                            m_l1 = __ballot_sync(0xffffffffu, l1);
                            m_b = __ballot_sync(0xffffffffu, act && b1 != 0.0f);
                            m_rb = __ballot_sync(0xffffffffu, act && rb[u] != 0.0f);
                        }
                        if(lane == 0)
                        {
                            WChunkTick *ct = &s_cnt[par][jj[u]];
                            if(m_l0)
                                atomicAdd(&ct->leave0, __popc(m_l0));
                            if(m_a)
                                atomicAdd(&ct->in_db0, __popc(m_a));
                            if(m_ra)
                                atomicAdd(&ct->in_raw0, __popc(m_ra));
                            if(TWO)
                            {
                                if(m_l1)
                                    atomicAdd(&ct->leave1, __popc(m_l1));
                                if(m_b)
                                    atomicAdd(&ct->in1, __popc(m_b));
                                if(m_rb)
                                    atomicAdd(&ct->in_raw1, __popc(m_rb));
                            }
                        }
                    }
                }
            }
            __syncthreads();
            // phase 2: the silent rule per tick (:341-356; with m_last_silent assigned on every path it reduces to "no
            // channel has a non-zero entry"), uniform over the CTA
            // Lane l evaluates tick l: the window count before its test is the count at chunk start plus the (entering -
            // leaving) sums of the ticks before it, minus what leaves with it.
            int Kc = K;
            bool hit = false;
            {
                WChunkTick ct{0, 0, 0, 0, 0, 0};
                if(lane < K)
                    ct = s_cnt[par][lane];
                int s0 = ct.in_db0 - ct.leave0, s1 = ct.in1 - ct.leave1;
#pragma unroll
                for(int o = 1; o < 32; o <<= 1)
                {
                    const int v0 = __shfl_up_sync(0xffffffffu, s0, o), v1 = __shfl_up_sync(0xffffffffu, s1, o);
                    s0 += (lane >= o) ? v0 : 0;
                    if(TWO)
                        s1 += (lane >= o) ? v1 : 0;
                }
                bool any = (wc0 + s0 - ct.in_db0 > 0) || (ct.in_raw0 > 0);
                if(MODE == 2)
                    any = any || (wc1 + s1 - ct.in1 > 0) || (ct.in_raw1 > 0);
                if(MODE == 1)
                    any = any || (wc1 + s1 > 0); // raw buffer: the tick's own points are part of what is tested
                const unsigned silent_mask = __ballot_sync(0xffffffffu, lane < K && !any);
                if(silent_mask != 0)
                {
                    hit = true;
                    Kc = __ffs(silent_mask);
                }
                // counts after the last processed tick (the DB_MIN fill below overrides the display channels after a hit)
                wc0 += __shfl_sync(0xffffffffu, s0, Kc - 1);
                if(TWO)
                    wc1 += __shfl_sync(0xffffffffu, s1, Kc - 1);
            }
            // rows of ticks [t, t+Kc): windows of E in time order (without `out`, MODE 3 still walks them for the state row)
            const bool wr_out = !DISP || p.out != nullptr;
            if(wr_out || MODE == 3)
            {
                const bool wr_state1 = (MODE == 3) && (t + Kc == p.n_ticks);
                if(vec)
                {
                    // one float4 of a row per thread and step; the silent row (at most the last one) is a constant
                    const int W4 = W >> 2, per = DCH * W4, rows = Kc - (hit ? 1 : 0), total = rows * per;
                    const unsigned magic = 0xffffffffu / (unsigned)per + 1u; // it / per == umulhi(it, magic) for it * per < 2^32
                    for(int it = tid; it < total; it += nt)
                    {
                        const int j = (int)__umulhi((unsigned)it, magic), r = it - j * per, d = (DCH == 2) ? (r >= W4) : 0,
                                  i = (r - d * W4) * 4;
                        const int o1 = s_off[j + 1];
                        float e[4];
                        if(MODE == 3 && d == 1)
                        {
                            const int lim = W + s_off[j];
#pragma unroll
                            for(int k = 0; k < 4; ++k)
                            {
                                const int rel = o1 + i + k;
                                e[k] = (rel < lim) ? E0[wrap2(base + rel, CAP)] : N0[rel - W];
                            }
                        }
                        else
                        {
                            const float *Ed = (DCH == 2 && d == 1) ? E1 : E0;
                            const int start = wrap2(base + o1 + i, CAP);
                            if(start + 3 < CAP)
                            {
#pragma unroll
                                for(int k = 0; k < 4; ++k)
                                    e[k] = Ed[start + k];
                            }
                            else
                            {
#pragma unroll
                                for(int k = 0; k < 4; ++k)
                                    e[k] = Ed[wrap2(start + k, CAP)];
                            }
                        }
                        const float4 v = make_float4(e[0], e[1], e[2], e[3]);
                        if(wr_out)
                            __stcs(reinterpret_cast<float4 *>(p.out + (((size_t)s * p.n_ticks + t + j) * DCH + d) * W + i), v);
                        if(wr_state1 && d == 1 && j == Kc - 1)
                            *reinterpret_cast<float4 *>(st1 + i) = v;
                    }
                    if(hit)
                    {
                        const float4 v = make_float4(p.db_min, p.db_min, p.db_min, p.db_min);
                        float4 *orow = reinterpret_cast<float4 *>(p.out + ((size_t)s * p.n_ticks + t + Kc - 1) * DCH * W);
                        for(int it = tid; it < per; it += nt)
                        {
                            if(wr_out)
                                __stcs(orow + it, v);
                            if(wr_state1 && it >= W4)
                                reinterpret_cast<float4 *>(st1)[it - W4] = v;
                        }
                    }
                }
                else
                {
                    const int per = DCH * W, total = Kc * per;
                    for(int it = tid; it < total; it += nt)
                    {
                        const int j = it / per, r = it - j * per, d = (DCH == 2) ? (r >= W) : 0, i = r - d * W;
                        const bool sil = hit && (j == Kc - 1);
                        float v = p.db_min;
                        if(!sil)
                        {
                            const int rel = s_off[j + 1] + i;
                            if(MODE == 3 && d == 1)
                                v = (rel < W + s_off[j]) ? E0[wrap2(base + rel, CAP)] : N0[rel - W];
                            else
                                v = ((d == 0) ? E0 : E1)[wrap2(base + rel, CAP)];
                        }
                        if(wr_out)
                            __stcs(p.out + (((size_t)s * p.n_ticks + t + j) * DCH + d) * W + i, v);
                        if(wr_state1 && d == 1 && j == Kc - 1)
                            st1[i] = v;
                    }
                }
                if(!DISP && p.out_silent != nullptr && tid < Kc)
                    p.out_silent[(size_t)s * p.n_ticks + t + tid] = (hit && tid == Kc - 1) ? 1 : 0;
            }
            if constexpr(DISP)
            {
                if(p.out_silent != nullptr && tid < Kc)
                    p.out_silent[(size_t)s * p.n_ticks + t + tid] = (hit && tid == Kc - 1) ? 1 : 0;
                // the same windows of E (the silent row, at most the last one, is DB_MIN in the display channels)
                __shared__ unsigned long long s_min[WCH_KMAX];
                const int b0 = base, silent_j = hit ? Kc - 1 : -1;
                wave_display(
                    p,
                    [&](int j, int d) {
                        const int o1 = s_off[j + 1];
                        const float *a = (DCH == 2 && MODE != 3 && d == 1) ? E1 : E0;
                        if(MODE == 3 && d == 1)
                            return RowSeg{a, N0 + (o1 - W), wrap2(b0 + o1, CAP), CAP, W + s_off[j] - o1, j == silent_j, p.db_min};
                        return RowSeg{a, a, wrap2(b0 + o1, CAP), CAP, W, j == silent_j, p.db_min};
                    },
                    s, t, Kc, wsm + p.scratch_off, s_min, tid, nt);
            }
            last_silent = hit;
            if(hit)
            {
                // :360-366: the display channels become DB_MIN; the ticks after it start from that buffer
                __syncthreads();
                base = wrap2(base + s_off[Kc], CAP);
                for(int i = tid; i < W; i += nt)
                {
                    E0[wrap2(base + i, CAP)] = p.db_min;
                    if(MODE == 2)
                        E1[wrap2(base + i, CAP)] = p.db_min;
                }
                wc0 = W;
                if(MODE == 2)
                    wc1 = W;
                if(tid < WCH_KMAX)
                    s_cnt[par][tid] = WChunkTick{0, 0, 0, 0, 0, 0};
                t += Kc;
            }
            else
            {
                base = wrap2(base + C, CAP);
                t += K;
                par ^= 1;
            }
            __syncthreads();
        }
        for(int i = tid; i < W; i += nt)
        {
            st0[i] = E0[wrap2(base + i, CAP)];
            if(TWO)
                st1[i] = E1[wrap2(base + i, CAP)];
        }
        if(tid == 0)
            p.flags[s] = last_silent ? 1 : 0;
        __syncthreads();
    }
}

// hidden / capture-timeout branch (src/source_generic.cpp:280-289)
__global__ void wave_reset_kernel(float *state, unsigned char *flags, int n_streams, int dch, int W, float db_min)
{
    for(int s = blockIdx.x; s < n_streams; s += gridDim.x)
    {
        if(flags[s] != 0)
            continue;
        for(int i = threadIdx.x; i < dch * W; i += blockDim.x)
            state[(size_t)s * 2 * W + i] = db_min;
        __syncthreads();
        if(threadIdx.x == 0)
            flags[s] = 1;
    }
}

// wf_wave_get_state / wf_wave_set_state: the state of streams [first, first+count) between the device layouts and the
// sections of one staging buffer (x_*, null = skipped), one CTA per stream.  Rows d < och of the [2][width] scrolling
// buffers (row 1 of a one-channel engine shown as one is never used).
struct WStateIO {
    float *state, *hold;
    unsigned char *flags;
    float *x_db, *x_hold;    // [count][och][width], [count][cc][D]
    unsigned char *x_flags;  // [count]
    int first, count, och, width, cc, D;
};
template<bool SET>
__global__ void wave_state_kernel(const WStateIO q)
{
    for(int i = blockIdx.x; i < q.count; i += gridDim.x)
    {
        const int s = q.first + i;
        if(q.x_db)
            for(int k = threadIdx.x; k < q.och * q.width; k += blockDim.x)
            {
                float *d = q.state + (size_t)s * 2 * q.width + k, *x = q.x_db + (size_t)i * q.och * q.width + k;
                if(SET)
                    *d = *x;
                else
                    *x = *d;
            }
        if(q.x_hold)
        {
            const long long n = (long long)q.cc * q.D;
            for(long long k = threadIdx.x; k < n; k += blockDim.x)
            {
                float *d = q.hold + (size_t)s * n + k, *x = q.x_hold + (size_t)i * n + k;
                if(SET)
                    *d = *x;
                else
                    *x = *d;
            }
        }
        if(q.x_flags && threadIdx.x == 0)
        {
            if(SET)
                q.flags[s] = q.x_flags[i] & 1;
            else
                q.x_flags[i] = q.flags[s] & 1;
        }
    }
}

// util.hpp's audio_frames_to_ns / ns_to_audio_frames (128-bit multiply-divide).  The 64-bit form is the same quotient
// whenever the product fits, which it does for everything but multi-day spans; the 128-bit division costs ~50 ns and the
// plan evaluates one per point.
__host__ __device__ inline uint64_t frames_to_ns(uint64_t sr, uint64_t frames)
{
    if(frames <= UINT64_MAX / 1000000000ull)
        return (frames * 1000000000ull) / sr;
    return (uint64_t)(((unsigned __int128)frames * 1000000000ull) / sr);
}
__host__ __device__ inline uint64_t ns_to_frames(uint64_t sr, uint64_t ns)
{
    if(ns <= UINT64_MAX / sr)
        return (ns * sr) / 1000000000ull;
    return (uint64_t)(((unsigned __int128)ns * sr) / 1000000000ull);
}

// ---- the tick plan: the timestamp walk of tick_waveform, shared by the host (plan_ticks) and the device (wave_plan_kernel) ----
// The clock the reference derives from packet timestamps, carried from call to call (on the host, or in wf_wave::d_clock for
// an engine created with device_clock = 1).  `buffered`: samples in the plugin's capture buffer after the last tick.
struct WaveClock {
    uint64_t clock, audio_ts, waveform_ts, buffered;
};
constexpr uint64_t kClockStart = 10ull * 1000000000ull; // the capture clock of a new engine, in ns (10 s)
// What a call's walk depends on besides the clock: the config, the sync offset's D and the call's hop (wave_walk).
struct WaveWalk {
    uint64_t sr, ws, D, width, step_ns, hop, hop_ns, D_ns;
    uint64_t span_ns;      // width * step_ns (< 2^53: at most meter_ms * 10^6)
    double inv_step;       // 1 / step_ns, for the quotient estimate of wave_tick
    uint64_t ss_total, ss_total_ns; // the buffer a tick sees after one that emitted (min(D + hop, ws + D)) and its span in ns
};
// One tick of the plan: it emits `count` points, point i at timestamp ts0 + i * step_ns, from a buffer of `total` samples
// whose newest ends at audio_ts.
struct WaveTick {
    uint64_t ts0, audio_ts, total;
    uint32_t count, pad;
};

WaveWalk wave_walk(const wf_wave_config &c, uint64_t ws, uint64_t D, int hop)
{
    WaveWalk k{};
    k.sr = c.sample_rate;
    k.ws = ws;
    k.D = D;
    k.width = (uint64_t)c.width;
    k.step_ns = ((uint64_t)c.meter_ms * 1000000ull) / k.width; // :303
    k.hop = (uint64_t)hop;
    k.hop_ns = frames_to_ns(k.sr, k.hop);
    k.D_ns = frames_to_ns(k.sr, D);
    k.span_ns = k.width * k.step_ns;
    k.inv_step = 1.0 / (double)k.step_ns;
    k.ss_total = std::min(D + k.hop, ws + D);
    k.ss_total_ns = frames_to_ns(k.sr, k.ss_total);
    return k;
}

// One tick of tick_waveform (src/source_generic.cpp:290-339,358) for a packet of `hop` samples that ends "now", with the sync
// offset's reserve of D samples; advances `c`.
//
// The reference emits points in a loop, i = 0, 1, ... < width, that stops at the first i with  ts >= stop_ts  or  ts <
// waveform_ts,  ts = waveform_ts + i * step_ns (mod 2^64).  The count is computed in closed form instead:
//   - i * step_ns < width * step_ns <= meter_ms * 10^6 never overflows, so ts only wraps when the sum exceeds 2^64 - 1;
//   - without a wrap ts grows with i, so "ts < stop_ts" holds for a prefix of i: the first ceil((stop_ts - waveform_ts) /
//     step_ns) values when waveform_ts < stop_ts, none otherwise;
//   - every ts of that prefix is below stop_ts <= 2^64 - 1, so none of them wraps: the wrap test never ends the loop first.
// Hence count = min(width, ceil((stop_ts - waveform_ts) / step_ns)), 0 when waveform_ts >= stop_ts.  The quotient is needed
// only below width, where the difference is below span_ns < 2^53: a double estimate (within 1 of the quotient) corrected by
// exact integer products gives it without a 64-bit division.
__host__ __device__ inline WaveTick wave_tick(WaveClock &c, const WaveWalk &k)
{
    c.clock += k.hop_ns;
    c.audio_ts = c.clock; // timestamp + audio_len, src/source.cpp:1836
    // the buffer keeps m_waveform_samples + D samples (src/source.cpp:1881-1884, src/source_generic.cpp:310-311)
    const uint64_t total = (c.buffered + k.hop < k.ws + k.D) ? c.buffered + k.hop : k.ws + k.D;
    c.buffered = total;
    WaveTick tk{0, c.audio_ts, total, 0, 0};
    if(total <= k.D) // not enough audio in advance: no points, the clock stays (:296-298)
        return tk;
    const uint64_t total_ns = (total == k.ss_total) ? k.ss_total_ns : frames_to_ns(k.sr, total);
    const uint64_t start_ts = c.audio_ts - total_ns, stop_ts = c.audio_ts - k.D_ns;
    if((start_ts >= c.audio_ts) || (stop_ts > c.audio_ts)) // :321-322 (rollover guard)
        return tk;
    if(c.waveform_ts < start_ts)
        c.waveform_ts = start_ts; // :323-324 (catch-up)
    if((c.waveform_ts > stop_ts) && ((c.waveform_ts - stop_ts) > k.step_ns))
        c.waveform_ts = start_ts; // :325-326 (desync)
    uint64_t count = 0;
    if(c.waveform_ts < stop_ts)
    {
        const uint64_t d = stop_ts - c.waveform_ts;
        if(d >= k.span_ns)
            count = k.width;
        else
        {
            count = (uint64_t)((double)d * k.inv_step); // the floor of the quotient, or one off either way
            while(count * k.step_ns < d)
                ++count;
            while(count > 0 && (count - 1) * k.step_ns >= d)
                --count;
        }
    }
    tk.ts0 = c.waveform_ts;
    tk.count = (uint32_t)count;
    c.waveform_ts += count * k.step_ns; // :358
    c.buffered = k.D;                   // consumed all but the reserve (:327)
    return tk;
}

// The source of point i of tick t: its sample (:336) as an index into  holdback(D) ++ the call's PCM,  minus `base`, or -1
// for a start-up zero.  The packet of tick t ends at D + (t+1)*hop there.
__host__ __device__ inline int wave_point_src(const WaveWalk &k, const WaveTick &tk, uint64_t i, int t, long long base)
{
    const uint64_t ts = tk.ts0 + i * k.step_ns;
    uint64_t index = ns_to_frames(k.sr, tk.audio_ts - ts);
    index = (index < k.D + 1) ? k.D + 1 : ((index > tk.total) ? tk.total : index);
    const long long pos = (long long)k.D + (long long)(t + 1) * (long long)k.hop - (long long)index - base;
    return pos < 0 ? -1 : (int)pos;
}

// Steady-state runs of the walk.  A tick that starts with buffered == D sees a buffer of ss_total samples.  If it passes the
// rollover guard, neither catches up nor resets, and emits no more than width points, it ends with buffered == D again, and
// its points continue the lattice waveform_ts + i * step_ns of the tick before.  So from a state c0 with buffered == D, as
// long as that holds, tick j of the run (j = 0, 1, ...) has
//   audio_ts = c0.clock + (j+1) * hop_ns,  stop_ts = audio_ts - D_ns,  start_ts = audio_ts - ss_total_ns,
//   the points of the lattice w0 + i * step_ns (w0 = c0.waveform_ts) with i in [K(stop of tick j-1), K(stop_ts)),
// where K(x) counts the lattice points below x (K := 0 for the tick before the run), and every tick can be evaluated on its
// own.  Why that is wave_tick's result: if the clock does not wrap, stop_ts grows with j, so K does not decrease; the tick
// enters with waveform_ts = W = w0 + K_in * step_ns; wave_tick's count is ceil((stop_ts - W) / step_ns) = K(stop_ts) - K_in
// when W < stop_ts, and 0 when W >= stop_ts (then K_in >= K(stop_ts) >= K_in); it leaves waveform_ts = w0 + K(stop_ts) *
// step_ns either way.  run_tick returns false where a condition of that argument fails (a wrap of the clock or of W, the
// guard, a catch-up, a reset, more than width points, or ss_total <= D); the walk then takes that tick with wave_tick.
__device__ __forceinline__ uint64_t lattice_below(uint64_t x, uint64_t w0, uint64_t step)
{
    return (x > w0) ? (x - w0 - 1) / step + 1 : 0;
}
__device__ __forceinline__ bool run_tick(const WaveClock &c0, const WaveWalk &k, uint64_t j, WaveTick &tk, WaveClock &out)
{
    if(k.ss_total <= k.D || __umul64hi(j + 1, k.hop_ns) != 0 || (j + 1) * k.hop_ns > UINT64_MAX - c0.clock)
        return false;
    const uint64_t audio = c0.clock + (j + 1) * k.hop_ns, start = audio - k.ss_total_ns, stop = audio - k.D_ns;
    if((start >= audio) || (stop > audio))
        return false;
    const uint64_t w0 = c0.waveform_ts;
    // the stop of tick j-1: only used when that tick passed the guard too (else the run ends before tick j)
    const uint64_t kin = (j == 0) ? 0 : lattice_below(stop - k.hop_ns, w0, k.step_ns);
    const uint64_t kout = lattice_below(stop, w0, k.step_ns);
    if(kout < kin || kout - kin > k.width || __umul64hi(kin, k.step_ns) != 0 || kin * k.step_ns > UINT64_MAX - w0)
        return false;
    const uint64_t W = w0 + kin * k.step_ns;
    if((W < start) || ((W > stop) && (W - stop > k.step_ns)))
        return false;
    tk = WaveTick{W, audio, k.ss_total, (uint32_t)(kout - kin), 0};
    out = WaveClock{audio, audio, W + (kout - kin) * k.step_ns, k.D};
    return true;
}

// The device planner of a device-clock engine: the plan of one call, in the layout plan_ticks writes with base = 0.  One
// CTA.  (1) The walk: while the clock is in a steady state (buffered == D) the CTA evaluates up to kPlanThreads ticks of the
// run at once (run_tick, a thread per tick) and keeps them up to the first that breaks the run; thread 0 takes that tick
// and every tick outside a run (the start-up, a catch-up) with wave_tick.  (2) off[] as a prefix sum of the counts.  (3)
// Every warp fills the sources of its ticks' points.  Packets end "now", so stop_ts never decreases and no clock comes near
// 2^64 ns: the rollover guard and the desync reset cannot fire here, and are kept only so that the walk is plan_ticks' own.
constexpr int kPlanThreads = 1024;
__global__ void __launch_bounds__(kPlanThreads) wave_plan_kernel(WaveClock *clk, const WaveWalk k, int n_ticks, int *off,
                                                                 int *src, WaveTick *ticks)
{
    __shared__ WaveClock s_c;
    __shared__ int s_t, s_bad, s_carry;
    __shared__ int s_warp[kPlanThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if(tid == 0)
    {
        s_c = *clk;
        s_t = 0;
        s_carry = 0;
        off[0] = 0;
    }
    __syncthreads();
    for(;;)
    {
        const int t = s_t;
        const bool steady = s_c.buffered == k.D;
        const WaveClock c0 = s_c;
        __syncthreads();
        if(t >= n_ticks)
            break;
        if(steady)
        {
            const int n = min(n_ticks - t, kPlanThreads);
            if(tid == 0)
                s_bad = n;
            __syncthreads();
            WaveTick tk;
            WaveClock ex;
            const bool ok = tid < n && run_tick(c0, k, (uint64_t)tid, tk, ex);
            if(tid < n && !ok)
                atomicMin(&s_bad, tid);
            __syncthreads();
            const int bad = s_bad;
            if(ok && tid < bad)
                ticks[t + tid] = tk;
            if(ok && tid == bad - 1)
                s_c = ex;
            __syncthreads();
            if(tid == 0)
            {
                int u = t + bad;
                if(bad < n)
                {
                    // the tick that ends the run; when it is the run's first (a catch-up at every tick, say), a stretch
                    // of ticks, so that such calls do not pay an attempt per tick
                    WaveClock c = s_c;
                    for(int q = 0; q < ((bad == 0) ? 64 : 1) && u < n_ticks; ++q)
                        ticks[u++] = wave_tick(c, k);
                    s_c = c;
                }
                s_t = u;
            }
        }
        else if(tid == 0)
        {
            WaveClock c = s_c;
            int u = t;
            do
                ticks[u++] = wave_tick(c, k);
            while(u < n_ticks && c.buffered != k.D);
            s_c = c;
            s_t = u;
        }
        __syncthreads();
    }
    if(tid == 0)
        *clk = s_c;
    for(int base = 0; base < n_ticks; base += kPlanThreads)
    {
        const int u = base + tid;
        int v = (u < n_ticks) ? (int)ticks[u].count : 0;
#pragma unroll
        for(int o = 1; o < 32; o <<= 1)
        {
            const int x = __shfl_up_sync(0xffffffffu, v, o);
            v += (lane >= o) ? x : 0;
        }
        if(lane == 31)
            s_warp[warp] = v;
        __syncthreads();
        if(warp == 0)
        {
            int x = s_warp[lane];
#pragma unroll
            for(int o = 1; o < 32; o <<= 1)
            {
                const int y = __shfl_up_sync(0xffffffffu, x, o);
                x += (lane >= o) ? y : 0;
            }
            s_warp[lane] = x;
        }
        __syncthreads();
        const int incl = s_carry + v + (warp ? s_warp[warp - 1] : 0);
        if(u < n_ticks)
            off[u + 1] = incl;
        __syncthreads();
        if(tid == kPlanThreads - 1)
            s_carry = incl;
        __syncthreads();
    }
    for(int t = warp; t < n_ticks; t += kPlanThreads / 32)
    {
        const WaveTick tk = ticks[t];
        int *s = src + off[t];
        for(uint32_t i = lane; i < tk.count; i += 32)
            s[i] = wave_point_src(k, tk, i, t, 0);
    }
}

} // namespace

struct wf_wave : wf::HostCore {
    wf_wave_config cfg{};
    int dch = 1, och = 1;
    size_t ws = 0;        // m_waveform_samples
    float db_min = 0.0f;
    // the clock the reference derives from packet timestamps (shared by all streams: they tick together); `buffered` holds
    // the start-up zeros at first (src/source.cpp:1243-1248), then at most D (tick_waveform keeps the reserve)
    WaveClock clk{kClockStart, 0, 0, 0};
    int D = 0;            // samples the audio sync offset reserves (wf_wave_config.sync_offset_ms)
    // device_clock of wf_wave_create_with_clock: the clock lives in d_clock (created as clk is), and wave_plan_kernel plans
    // every call from it
    bool dev_clock = false;
    wf::DevBuf<WaveClock> d_clock;
    wf::DevBuf<WaveTick> d_ticks; // [n_ticks] of the call: wave_plan_kernel's per-tick walk results
    wf::DevBuf<float> d_hold;   // [max_streams][cc][D]: the last D samples of each stream and channel, zeros at creation
    wf::DevBuf<float> s_window; // holdback ++ new of a call, in its sample type (counts floats)
    wf::DevBuf<float> d_state;
    wf::DevBuf<unsigned char> d_flags;
    wf::DevBuf<int> d_src, d_off;
    wf::DevBuf<float> s_pcm, s_out, s_rms, s_points, s_pixels, s_min;
    wf::DevBuf<unsigned char> s_silent;
    // wf_wave_get_state / wf_wave_set_state: the sections of a call, on the device and on the host
    wf::DevBuf<unsigned char> s_state;
    std::vector<unsigned char> h_state;
    struct PlanSlot {
        int *h = nullptr; // pinned: off[] then src[]
        size_t cap = 0;
        cudaEvent_t done = nullptr;
        bool used = false;
        ~PlanSlot()
        {
            if(h)
                cudaFreeHost(h);
            if(done)
                cudaEventDestroy(done);
        }
    };
    static constexpr int kSlots = 4;
    PlanSlot slots[kSlots];
    int slot_next = 0;
    cudaStream_t last_stream = nullptr;
    // The kernel of a call, [display outputs][s16]: wave_chunk_kernel of the engine's channel layout, or with WF_WAVE_CHUNK=0
    // the per-tick wave_kernel (kept for A/B and bit-identity tests).  The display entries exist with display settings only.
    struct TickLaunch {
        const void *kernel = nullptr;
        size_t smem = 0; // dynamic shared memory before the Gaussian's scratch rows
        int per_sm = 0;  // resident CTAs per SM: the grid is at most one wave of them
    } tick[2][2];
    // display stage: only when the config carried display settings (current struct size) and width >= 2
    bool display = false;
    wf::Tables tab;
    wf::DevBuf<float> d_tab;      // interp weights | interp indices | Gaussian
    int disp_scratch = 0;         // floats of Gaussian scratch (dch * width, or 0 without the filter)
};

namespace {

thread_local std::string g_wave_create_error;

// A config is the current struct, the previous one (which ends before sync_offset_ms: no offset) or the one before, which
// ends before interp_mode: its display settings are absent.
constexpr size_t kPrevWaveConfig = offsetof(wf_wave_config, interp_mode);
constexpr size_t kSyncWaveConfig = offsetof(wf_wave_config, sync_offset_ms);

// accept_struct for a wave config; `display_settings`: the caller's struct carries them
bool accept_wave_config(const wf_wave_config *in, wf_wave_config &out, bool *display_settings = nullptr)
{
    if(!wf::accept_struct(in, {kSyncWaveConfig, kPrevWaveConfig}, out))
        return false;
    if(display_settings)
        *display_settings = in->struct_size != kPrevWaveConfig;
    return true;
}

// The limits of a waveform config that the clock and the buffers depend on (wf_wave_create, the previews): width in
// [1, 8192] and a nanosecond step meter_ms * 10^6 / width of at least 1.
bool wave_clock_ok(const wf_wave_config &c)
{
    return c.sample_rate >= 1 && c.width >= 1 && c.width <= 8192 && c.meter_ms >= 1 &&
           ((uint64_t)c.meter_ms * 1000000ull) / (uint64_t)c.width != 0 && wf::sync_offset_ok(c.sync_offset_ms);
}

// The tick kernel for parameters P and sample type TS: the chunk kernel of channel layout `mode`, or the per-tick kernel
template<class P, typename TS>
const void *tick_kernel(bool chunked, int mode)
{
    static const void *const chunk[4] = {(const void *)wave_chunk_kernel<0, P, TS>, (const void *)wave_chunk_kernel<1, P, TS>,
                                         (const void *)wave_chunk_kernel<2, P, TS>, (const void *)wave_chunk_kernel<3, P, TS>};
    return chunked ? chunk[mode] : (const void *)wave_kernel<P, TS>;
}

// The tick-by-tick timestamp walk of tick_waveform for packets of `hop` samples that end "now" (wave_tick), on the host
// clock: appends, per tick, the source sample of every new point as an index into  holdback(D) ++ the call's PCM,  minus
// `base`; an index below 0 stands for a start-up zero and is -1.
void plan_ticks(wf_wave *w, int n_ticks, int hop, long long base, std::vector<int> &src, std::vector<int> &off)
{
    const WaveWalk k = wave_walk(w->cfg, w->ws, (uint64_t)w->D, hop);
    src.clear();
    off.assign(1, 0);
    for(int t = 0; t < n_ticks; ++t)
    {
        const WaveTick tk = wave_tick(w->clk, k);
        for(uint32_t i = 0; i < tk.count; ++i)
            src.push_back(wave_point_src(k, tk, i, t, base));
        off.push_back((int)src.size());
    }
}

// The plan of a call on the host clock (plan_ticks), uploaded to d_off / d_src on `st`.  The plan is a host walk of the
// nanosecond clock, so a replay would repeat this call's plan instead of advancing the clock: a call on a capturing stream
// is refused before anything is enqueued or advanced, and the capture stays valid.
int upload_host_plan(wf_wave *w, cudaStream_t st, int n_ticks, int hop)
{
    cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
    WF_CHECK(w, cudaStreamIsCapturing(st, &capture));
    if(capture != cudaStreamCaptureStatusNone)
        return wf::fail(w, WF_ERR_INVALID_ARG, "the waveform engine cannot be captured into a CUDA graph: its tick plan is "
                                               "walked on the host from the engine's clock at every call (create the engine "
                                               "with device_clock = 1)");
    std::vector<int> src, off;
    plan_ticks(w, n_ticks, hop, 0, src, off);
    int rc;
    if((rc = w->d_src.reserve(w, std::max<size_t>(1, src.size()))))
        return rc;
    if((rc = w->d_off.reserve(w, off.size())))
        return rc;
    // the plan goes through one of a few pinned slots, so a call neither waits for the previous kernel nor leaves the
    // device reading a vector that is about to go away; a slot is reused only after its copy has completed
    wf_wave::PlanSlot &ps = w->slots[w->slot_next];
    w->slot_next = (w->slot_next + 1) % wf_wave::kSlots;
    if(ps.used)
        WF_CHECK(w, cudaEventSynchronize(ps.done));
    const size_t need = src.size() + off.size();
    if(need > ps.cap)
    {
        if(ps.h)
            cudaFreeHost(ps.h);
        ps.h = nullptr;
        ps.cap = 0;
        WF_CHECK(w, cudaMallocHost((void **)&ps.h, need * sizeof(int)));
        ps.cap = need;
    }
    if(!ps.done)
        WF_CHECK(w, cudaEventCreateWithFlags(&ps.done, cudaEventDisableTiming));
    memcpy(ps.h, off.data(), off.size() * sizeof(int));
    if(!src.empty())
        memcpy(ps.h + off.size(), src.data(), src.size() * sizeof(int));
    if(w->last_stream != nullptr && w->last_stream != st)
        WF_CHECK(w, cudaStreamSynchronize(w->last_stream)); // d_src / d_off may still be read by a call on another stream
    w->last_stream = st;
    WF_CHECK(w, cudaMemcpyAsync(w->d_off, ps.h, off.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    if(!src.empty())
        WF_CHECK(w, cudaMemcpyAsync(w->d_src, ps.h + off.size(), src.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WF_CHECK(w, cudaEventRecord(ps.done, st));
    ps.used = true;
    return WF_OK;
}

} // namespace

extern "C" {

void wf_wave_config_init(wf_wave_config *c)
{
    memset(c, 0, sizeof(*c));
    c->struct_size = (uint32_t)sizeof(wf_wave_config);
    c->device = -1;
    c->max_streams = 1;
    c->sample_rate = 48000;
    c->capture_channels = 2;
    c->stereo = 0;
    c->width = 800;
    c->meter_ms = 150;
    c->normalize_volume = 0;
    c->volume_target = -8.0f;
    c->max_gain = 30.0f;
    c->interp_mode = WF_INTERP_CATROM;
    c->filter_mode = WF_FILTER_NONE;
    c->filter_radius = 1.5f;
    c->height = 225;
    c->floor_db = -65;
    c->ceiling_db = 0;
    c->channel_spacing = 0;
    c->sync_offset_ms = 0;
}

const char *wf_wave_last_error(const wf_wave *w) { return w ? w->last_error.c_str() : g_wave_create_error.c_str(); }

int wf_wave_create(const wf_wave_config *cfg_in, wf_wave **out) { return wf_wave_create_with_clock(cfg_in, 0, out); }

int wf_wave_create_with_clock(const wf_wave_config *cfg_in, int32_t device_clock, wf_wave **out)
{
    if(!cfg_in || !out)
        return WF_ERR_INVALID_ARG;
    *out = nullptr;
    return wf::create_engine(out, g_wave_create_error, wf_wave_destroy, [&](wf_wave *w) -> int {
        bool display_settings = false;
        if(!accept_wave_config(cfg_in, w->cfg, &display_settings))
            return wf::fail(w, WF_ERR_ABI, "wf_wave_config.struct_size mismatch");
        const wf_wave_config *cfg = &w->cfg;
        if(cfg->capture_channels < 1 || cfg->capture_channels > 2 || cfg->max_streams < 1 || !wave_clock_ok(*cfg))
            return wf::fail(w, WF_ERR_INVALID_ARG, "bad waveform config (or meter_ms too small for this width: a step of 0 ns, "
                                                   "or sync_offset_ms outside [-1000, 1000])");
        if(device_clock != 0 && device_clock != 1)
            return wf::fail(w, WF_ERR_INVALID_ARG, "device_clock must be 0 or 1");
        // the display tables are built only for a config that passed the checks above (width <= 8192)
        const bool display = display_settings && cfg->width >= 2;
        if(display)
        {
            const char *why = "bad display settings";
            if(wf::build_wave_tables(*cfg, w->tab, &why) != WF_OK)
                return wf::fail(w, WF_ERR_INVALID_ARG, "%s", why);
        }
        if(int rc = wf::open_device(w, cfg->device))
            return rc;
        w->dch = cfg->stereo ? 2 : 1;
        w->och = ((cfg->capture_channels > 1) || cfg->stereo) ? 2 : 1; // src/source.cpp:1171
        w->ws = (size_t)((double)cfg->sample_rate * ((double)cfg->meter_ms / 1000.0)); // :1141
        w->clk.buffered = (uint64_t)cfg->width;                                        // :1243-1248 (m_fft_size zeros)
        w->D = wf::sync_delay(cfg->sample_rate, cfg->sync_offset_ms);
        w->dev_clock = device_clock == 1;
        w->db_min = 20.0f * log10f(1.17549435e-38f);
        w->display = display;
        // the Gaussian's scratch rows follow the kernel's own shared memory in the DISP kernels
        w->disp_scratch = (display && w->tab.cfg.filter_mode == WF_FILTER_GAUSS) ? w->dch * cfg->width : 0;
        {
            const bool chunked = wf::env_flag("WF_WAVE_CHUNK", true), two = cfg->capture_channels > 1;
            const int mode = cfg->stereo ? (two ? 2 : 3) : (two ? 1 : 0); // the chunk kernel's channel layout
            static const int mult[4] = {2, 4, 4, 3};                       // its floats per point; the per-tick kernel's: 2
            const size_t smem = (size_t)(chunked ? mult[mode] : 2) * cfg->width * sizeof(float);
            const void *const kernels[2][2] = {
                {tick_kernel<WParams, float>(chunked, mode), tick_kernel<WParams, int16_t>(chunked, mode)},
                {tick_kernel<WDisp, float>(chunked, mode), tick_kernel<WDisp, int16_t>(chunked, mode)}};
            for(int disp = 0; disp < (display ? 2 : 1); ++disp)
            {
                int per_sm = 8;
                if(chunked)
                {
                    // the float kernel's occupancy sizes the grid of both (one resident wave: streams are equal work, a
                    // partial second wave is a tail); the query needs the shared-memory limit raised first
                    const size_t bytes = smem + (disp ? w->disp_scratch * sizeof(float) : 0);
                    WF_CHECK(w, wf::opt_in_smem(kernels[disp][0], w->device, bytes));
                    WF_CHECK(w, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernels[disp][0], 256, bytes));
                    per_sm = std::max(1, per_sm);
                }
                for(int s16 = 0; s16 < 2; ++s16)
                    w->tick[disp][s16] = {kernels[disp][s16], smem, per_sm};
            }
        }
        int rc;
        if(display)
        {
            const auto &t = w->tab;
            if((rc = w->d_tab.reserve(w, t.interp_indices.size() + t.interp_weights.size() + t.gauss.size())))
                return rc;
            float *q = w->d_tab;
            for(const auto *v : {&t.interp_weights, &t.interp_indices, &t.gauss}) // weights first: 16-byte aligned
            {
                if(!v->empty())
                    WF_CHECK(w, cudaMemcpy(q, v->data(), v->size() * sizeof(float), cudaMemcpyHostToDevice));
                q += v->size();
            }
        }
        const size_t S = (size_t)cfg->max_streams, n = S * 2 * (size_t)cfg->width;
        if((rc = w->d_state.reserve(w, n)))
            return rc;
        if((rc = w->d_flags.reserve(w, S)))
            return rc;
        WF_CHECK(w, cudaMemsetAsync(w->d_flags, 0, S, w->stream)); // m_last_silent := false, src/source.cpp:1236
        if(w->D > 0)
        {
            const size_t hold_n = S * cfg->capture_channels * (size_t)w->D;
            if((rc = w->d_hold.reserve(w, hold_n)))
                return rc;
            WF_CHECK(w, cudaMemsetAsync(w->d_hold, 0, hold_n * sizeof(float), w->stream));
        }
        if(w->dev_clock)
        {
            if((rc = w->d_clock.reserve(w, 1)))
                return rc;
            WF_CHECK(w, cudaMemcpy(w->d_clock.p, &w->clk, sizeof(WaveClock), cudaMemcpyHostToDevice));
        }
        if((rc = wf::fill_device(w, w->d_state, (long long)n, w->db_min, w->stream)))
            return rc;
        WF_CHECK(w, cudaStreamSynchronize(w->stream));
        return WF_OK;
    });
}

void wf_wave_destroy(wf_wave *w)
{
    if(!w)
        return;
    if(w->stream)
    {
        cudaSetDevice(w->device);
        cudaStreamSynchronize(w->stream);
        if(w->last_stream && w->last_stream != w->stream)
            cudaStreamSynchronize(w->last_stream);
    }
    delete w;
}

int wf_wave_process_async(wf_wave *w, const wf_wave_batch *b_in, void *cuda_stream)
{
    if(!w || !b_in)
        return WF_ERR_INVALID_ARG;
    wf::NvtxRange nvtx("wf_wave_process");
    // the current struct, the previous one (which ends before pcm_format: float PCM) or the one before (which ends before
    // out_points: no display outputs either)
    wf_wave_batch bv;
    if(!wf::accept_struct(b_in, {offsetof(wf_wave_batch, pcm_format), offsetof(wf_wave_batch, out_points)}, bv))
        return wf::fail(w, WF_ERR_ABI, "wf_wave_batch.struct_size %u != %zu", b_in->struct_size, sizeof(wf_wave_batch));
    const wf_wave_batch *b = &bv;
    if(b->n_ticks < 0 || b->hop < 1)
        return wf::fail(w, WF_ERR_INVALID_ARG, "n_ticks must be >= 0 and hop >= 1");
    if(b->n_streams != w->cfg.max_streams)
        return wf::fail(w, WF_ERR_CAPACITY, "a waveform call must tick all %d streams of the engine (got %d): the clock is shared",
                    w->cfg.max_streams, b->n_streams);
    const bool disp = b->out_points || b->out_pixels || b->out_min;
    if(disp && !w->display)
        return wf::fail(w, WF_ERR_INVALID_ARG, "display outputs need an engine created with display settings (and width >= 2)");
    if(b->n_ticks == 0)
        return WF_OK;
    if(!b->pcm || !(b->out || b->out_points || b->out_pixels))
        return wf::fail(w, WF_ERR_INVALID_ARG, "pcm is null, or none of out / out_points / out_pixels is set");
    wf::PcmBatch pb;
    if(int rc = wf::check_pcm_batch(w, *b, w->cfg.capture_channels, w->D, &pb))
        return rc;
    if(w->dev_clock && (long long)b->n_ticks * w->cfg.width > 0x7fffffffLL)
        return wf::fail(w, WF_ERR_INVALID_ARG, "n_ticks * width too large for one call");

    WF_CHECK(w, cudaSetDevice(w->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : w->stream;
    const int cc = w->cfg.capture_channels, W = w->cfg.width;
    const size_t S = (size_t)b->n_streams, T = (size_t)b->n_ticks;
    int rc;
    if(w->dev_clock)
    {
        // the plan is made on the device (wave_plan_kernel, launched below), so the call may be captured
        WF_CHECK(w, wf::begin_call(w, st));
        if((rc = wf::refuse_pageable(w, {b->pcm, b->input_rms, b->out, b->out_silent, b->out_points, b->out_pixels,
                                         b->out_min})))
            return rc;
        // a tick emits at most width points: the plan space of any clock
        if((rc = w->d_src.reserve(w, T * (size_t)W)))
            return rc;
        if((rc = w->d_off.reserve(w, T + 1)))
            return rc;
        if((rc = w->d_ticks.reserve(w, T)))
            return rc;
    }
    else if((rc = upload_host_plan(w, st, b->n_ticks, b->hop)))
        return rc;

    // a call with host buffers (told by pcm alone) is staged through device memory
    const size_t out_n = S * T * w->dch * (size_t)W;
    wf::Staging io(w, st, !wf::is_device_ptr(b->pcm));
    wf::PcmView pcm{io.in_bytes(w->s_pcm, b->pcm, pb.span * pb.sample_bytes), b->stream_stride, b->channel_stride};
    const float *d_rms = io.in(w->s_rms, b->input_rms, S * T);
    float *d_out = io.out(w->s_out, b->out, out_n);
    float *d_points = io.out(w->s_points, b->out_points, out_n);
    float *d_pixels = io.out(w->s_pixels, b->out_pixels, out_n);
    float *d_min = io.out(w->s_min, b->out_min, S * T * 2);
    unsigned char *d_silent = io.out(w->s_silent, b->out_silent, S * T);
    if(io.rc)
        return io.rc;
    WF_CHECK(w, wf::time_begin(w, st));
    // with a sync offset the plan indexes into holdback ++ new, and the holdback keeps the last D samples (wf_splice.hpp)
    if(w->D > 0)
    {
        const long long tl = (long long)T * b->hop;
        if((rc = wf::splice_holdback(w, w->d_hold, w->D, (int)S, cc, tl, w->D + tl, pb.s16, w->s_window, pcm, st)))
            return rc;
    }
    if(w->dev_clock)
    {
        const WaveWalk k = wave_walk(w->cfg, w->ws, (uint64_t)w->D, b->hop);
        WF_CHECK(w, wf::launch_kernel(wave_plan_kernel, w->device, 1, kPlanThreads, 0, st, {}, w->d_clock.p, k, b->n_ticks,
                                      w->d_off.p, w->d_src.p, w->d_ticks.p));
        w->launches++;
    }
    WParams p{};
    p.pcm = pcm.pcm;
    p.stream_stride = pcm.stream_stride;
    p.channel_stride = pcm.channel_stride;
    p.input_rms = d_rms;
    p.src = w->d_src;
    p.off = w->d_off;
    p.state = w->d_state;
    p.flags = w->d_flags;
    p.out = d_out;
    p.out_silent = d_silent;
    p.n_streams = b->n_streams;
    p.n_ticks = b->n_ticks;
    p.width = W;
    p.cc = cc;
    p.dch = w->dch;
    p.och = w->och;
    p.stereo = w->cfg.stereo;
    p.normalize = w->cfg.normalize_volume;
    p.vol_target = w->cfg.volume_target;
    p.max_gain = w->cfg.max_gain;
    p.db_min = w->db_min;
    const wf_wave::TickLaunch &l = w->tick[disp][pb.s16];
    WDisp pd{};
    if(disp)
    {
        const auto &t = w->tab;
        static_cast<WParams &>(pd) = p;
        pd.interp_w = t.interp_weights.empty() ? nullptr : w->d_tab.p;
        pd.interp_idx = w->d_tab + t.interp_weights.size();
        pd.gauss_w = t.gauss.empty() ? nullptr : w->d_tab + t.interp_weights.size() + t.interp_indices.size();
        pd.out_points = d_points;
        pd.out_pixels = d_pixels;
        pd.out_min = d_min;
        pd.taps = t.interp_taps;
        pd.filter = t.gauss.empty() ? 0 : 1;
        pd.gauss_radius = t.gauss_radius;
        pd.gauss_sum = t.gauss_sum;
        pd.ceiling_f = (float)t.cfg.ceiling_db;
        pd.dbrange_f = (float)(t.cfg.ceiling_db - t.cfg.floor_db);
        pd.px_hi = t.px_hi;
        pd.px_cpos = t.px_cpos;
        pd.scratch_off = (int)(l.smem / sizeof(float));
        pd.vec4 = ((W & 3) == 0) && ((reinterpret_cast<uintptr_t>(d_points) & 15) == 0) &&
                  ((reinterpret_cast<uintptr_t>(d_pixels) & 15) == 0);
    }
    const int grid = (int)std::min<size_t>(S, (size_t)w->sm_count * l.per_sm);
    const size_t scratch = disp ? (size_t)w->disp_scratch * sizeof(float) : 0;
    void *args[] = {disp ? (void *)&pd : (void *)&p};
    WF_CHECK(w, wf::launch_kernel(l.kernel, w->device, grid, 256, l.smem + scratch, st, {}, args));
    w->launches++;
    WF_CHECK(w, wf::time_end(w, st));
    return io.finish();
}

int wf_wave_process(wf_wave *w, const wf_wave_batch *b)
{
    int rc = wf_wave_process_async(w, b, nullptr);
    if(rc)
        return rc;
    WF_CHECK(w, cudaStreamSynchronize(w->stream));
    return WF_OK;
}

int wf_wave_reset(wf_wave *w)
{
    if(!w)
        return WF_ERR_INVALID_ARG;
    WF_CHECK(w, cudaSetDevice(w->device));
    WF_CHECK(w, wf::launch_kernel(wave_reset_kernel, w->device, std::min(w->cfg.max_streams, w->sm_count * 4), 256, 0,
                                  w->stream, {}, w->d_state.p, w->d_flags.p, w->cfg.max_streams, w->dch, w->cfg.width,
                                  w->db_min));
    w->launches++;
    WF_CHECK(w, cudaStreamSynchronize(w->stream));
    return WF_OK;
}

} // extern "C"

namespace {

static_assert(sizeof(wf_wave_clock) == sizeof(WaveClock) && offsetof(wf_wave_clock, clock_ns) == offsetof(WaveClock, clock) &&
                  offsetof(wf_wave_clock, audio_ts) == offsetof(WaveClock, audio_ts) &&
                  offsetof(wf_wave_clock, waveform_ts) == offsetof(WaveClock, waveform_ts) &&
                  offsetof(wf_wave_clock, buffered) == offsetof(WaveClock, buffered),
              "wf_wave_clock is WaveClock field for field");

// wf_wave_get_state (set = false) / wf_wave_set_state (set = true): the range check, then one copy and one launch on the
// engine's stream, which is synchronised
int wave_state(wf_wave *w, int32_t first, int32_t count, const float *db, const float *hold, const uint8_t *flags, bool set)
{
    if(!w)
        return WF_ERR_INVALID_ARG;
    if(int rc = wf::check_slot_range(w, first, count, w->cfg.max_streams, "state"))
        return rc;
    const size_t n = (size_t)count, cc = (size_t)w->cfg.capture_channels;
    wf::StateSections io;
    const int i_db = io.add(db, n * w->och * w->cfg.width * sizeof(float));
    const int i_hold = io.add(hold, n * cc * w->D * sizeof(float));
    const int i_flags = io.add(flags, n);
    if(io.empty())
        return WF_OK;
    WF_CHECK(w, cudaSetDevice(w->device));
    if(int rc = io.reserve(w, w->s_state, w->h_state))
        return rc;
    WStateIO q{};
    q.state = w->d_state;
    q.hold = w->d_hold;
    q.flags = w->d_flags;
    q.x_db = io.dev<float>(i_db);
    q.x_hold = io.dev<float>(i_hold);
    q.x_flags = io.dev<unsigned char>(i_flags);
    q.first = first;
    q.count = count;
    q.och = w->och;
    q.width = w->cfg.width;
    q.cc = (int)cc;
    q.D = w->D;
    const int grid = std::min(count, w->sm_count * 4);
    return io.run(w, w->stream, set, [&] {
        const cudaError_t err = wf::launch_kernel(set ? wave_state_kernel<true> : wave_state_kernel<false>, w->device,
                                                  grid, 256, 0, w->stream, {}, q);
        w->launches += (err == cudaSuccess);
        return err;
    });
}

// Whether the timestamp walk (wave_tick from the creation clock) can have left `c`; the rules are wf_wave_set_clock's in
// wfstft.h.  Before the first tick the clock is the creation clock.  Every tick advances the clock from kClockStart and
// sets audio_ts := clock; a tick that passes the rollover guard leaves buffered <= D (none emitted:
// the buffer, at most D; else the reserve D) and waveform_ts at most one step past its stop audio_ts - D_ns (the desync
// reset catches anything further); one stopped by the guard keeps its buffer (at most ws + D) and waveform_ts.
bool wave_clock_valid(const wf_wave *w, const WaveClock &c)
{
    const uint64_t width = (uint64_t)w->cfg.width, D = (uint64_t)w->D, sr = w->cfg.sample_rate;
    if(c.audio_ts == 0)
        return c.clock == kClockStart && c.waveform_ts == 0 && c.buffered == width;
    if(c.audio_ts != c.clock || c.clock < kClockStart)
        return false;
    if(c.buffered > std::max(width, D))
    {
        const uint64_t total_ns = frames_to_ns(sr, c.buffered), D_ns = frames_to_ns(sr, D);
        const bool guard = (c.audio_ts - total_ns >= c.audio_ts) || (c.audio_ts - D_ns > c.audio_ts);
        if(!guard || c.buffered > w->ws + D)
            return false;
    }
    const uint64_t step_ns = ((uint64_t)w->cfg.meter_ms * 1000000ull) / width;
    return (unsigned __int128)c.waveform_ts + frames_to_ns(sr, D) <= (unsigned __int128)c.audio_ts + step_ns;
}

} // namespace

extern "C" {

int wf_wave_get_state(wf_wave *w, int32_t first, int32_t count, float *db, float *hold, uint8_t *flags)
{
    return wave_state(w, first, count, db, hold, flags, false);
}

int wf_wave_set_state(wf_wave *w, int32_t first, int32_t count, const float *db, const float *hold, const uint8_t *flags)
{
    return wave_state(w, first, count, db, hold, flags, true);
}

int wf_wave_get_clock(wf_wave *w, wf_wave_clock *clk)
{
    if(!w || !clk)
        return WF_ERR_INVALID_ARG;
    WaveClock c = w->clk;
    if(w->dev_clock)
    {
        WF_CHECK(w, cudaSetDevice(w->device));
        WF_CHECK(w, cudaMemcpyAsync(&c, w->d_clock.p, sizeof(WaveClock), cudaMemcpyDeviceToHost, w->stream));
        WF_CHECK(w, cudaStreamSynchronize(w->stream));
    }
    memcpy(clk, &c, sizeof(c));
    return WF_OK;
}

int wf_wave_set_clock(wf_wave *w, const wf_wave_clock *clk)
{
    if(!w || !clk)
        return WF_ERR_INVALID_ARG;
    WaveClock c;
    memcpy(&c, clk, sizeof(c));
    if(!wave_clock_valid(w, c))
        return wf::fail(w, WF_ERR_INVALID_ARG,
                        "clock {%llu, %llu, %llu, %llu} cannot come from this engine's timestamp walk (see wfstft.h)",
                        (unsigned long long)c.clock, (unsigned long long)c.audio_ts, (unsigned long long)c.waveform_ts,
                        (unsigned long long)c.buffered);
    if(w->dev_clock)
    {
        WF_CHECK(w, cudaSetDevice(w->device));
        WF_CHECK(w, cudaMemcpyAsync(w->d_clock.p, &c, sizeof(WaveClock), cudaMemcpyHostToDevice, w->stream));
        WF_CHECK(w, cudaStreamSynchronize(w->stream));
    }
    else
        w->clk = c;
    return WF_OK;
}

int64_t wf_wave_preview_plan(const wf_wave_config *cfg_in, int32_t n_ticks, int32_t hop, int32_t *counts, int32_t *src,
                             int64_t capacity)
{
    if(!cfg_in || n_ticks < 0 || hop < 1)
        return WF_ERR_INVALID_ARG;
    wf_wave_config cfg_v;
    if(!accept_wave_config(cfg_in, cfg_v))
        return WF_ERR_ABI;
    const wf_wave_config *cfg = &cfg_v;
    if(!wave_clock_ok(*cfg))
        return WF_ERR_INVALID_ARG;
    wf_wave w; // host-only use: the same initial clock / start-up state wf_wave_create sets up
    w.cfg = *cfg;
    w.ws = (size_t)((double)cfg->sample_rate * ((double)cfg->meter_ms / 1000.0));
    w.clk.buffered = (uint64_t)cfg->width;
    w.D = wf::sync_delay(cfg->sample_rate, cfg->sync_offset_ms);
    std::vector<int> s, off;
    plan_ticks(&w, n_ticks, hop, w.D, s, off); // indices into the call's PCM: a first call's holdback is start-up zeros
    if(counts)
        for(int t = 0; t < n_ticks; ++t)
            counts[t] = off[t + 1] - off[t];
    if(src)
    {
        if((int64_t)s.size() > capacity)
            return WF_ERR_INVALID_ARG;
        memcpy(src, s.data(), s.size() * sizeof(int));
    }
    return (int64_t)s.size();
}

int64_t wf_wave_preview_table(const wf_wave_config *cfg_in, int which, float *out, int64_t capacity)
{
    if(!cfg_in)
        return WF_ERR_INVALID_ARG;
    wf_wave_config cfg;
    bool display_settings;
    if(!accept_wave_config(cfg_in, cfg, &display_settings))
        return WF_ERR_ABI;
    if(which != WF_TABLE_INTERP_INDICES && which != WF_TABLE_INTERP_WEIGHTS && which != WF_TABLE_GAUSS)
        return WF_ERR_INVALID_ARG;
    if(!wave_clock_ok(cfg)) // the limits wf_wave_create applies, before anything is sized by width
        return WF_ERR_INVALID_ARG;
    if(!display_settings)
        return 0; // an engine without display settings has no display tables
    wf::Tables t;
    const char *why = nullptr;
    if(int rc = wf::build_wave_tables(cfg, t, &why); rc != WF_OK)
        return rc;
    const std::vector<float> &v = (which == WF_TABLE_INTERP_INDICES) ? t.interp_indices
                                  : (which == WF_TABLE_INTERP_WEIGHTS) ? t.interp_weights
                                                                       : t.gauss;
    if(out)
    {
        if((int64_t)v.size() > capacity)
            return WF_ERR_INVALID_ARG;
        if(!v.empty())
            memcpy(out, v.data(), v.size() * sizeof(float));
    }
    return (int64_t)v.size();
}

int64_t wf_wave_launch_count(const wf_wave *w) { return w ? w->launches : 0; }

float wf_wave_last_kernel_ms(wf_wave *w) { return wf::last_kernel_ms(w); }

} // extern "C"
