// wf_wave.cu — waveform (oscilloscope) mode of the plugin (tick_waveform) as a batched sm_90a gather behind the C ABI of
// include/wfstft.h (wf_wave_*).  SURVEY.md §8(f) rank 4.
//
// Reference semantics restated (paths relative to the reference tree): src/source_generic.cpp:272-390 with the capture side
// of src/source.cpp:1817-1888 for packets that end "now"; setup src/source.cpp:1129-1143, :1181, :1243-1248.
//
// The reference walks a nanosecond clock: every tick it emits the points whose timestamps m_waveform_ts + i*step_ns fall
// into the span of the audio captured since the last tick and picks the NEAREST sample for each.  All of that arithmetic is
// independent of the audio itself, so the host plans a call once (plan_ticks: per tick the number of new points and, for
// each, which sample of the packet it takes — integer arithmetic, bit-exact) and the device does what is left per stream:
// gather the samples, keep the scrolling buffer (a ring in shared memory), evaluate the all-zero "silent" rule, convert
// the new points to dBFS (|x|, stereo / mono mix), add the volume compensation, and write the buffer row of every tick.
// HBM traffic: the packet's sectors once in, width floats per display channel and tick out.  There is no CPU fallback.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "wf_nvtx.hpp"
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

__device__ __forceinline__ float dbfs_dev(float mag, float db_min) { return (mag > 0.0f) ? 20.0f * log10f(mag) : db_min; }

// One CTA per stream; the scrolling buffers live in shared memory as rings (head = oldest point).
__global__ void __launch_bounds__(256) wave_kernel(const WParams p)
{
    extern __shared__ float ring[]; // [2][width]
    const int W = p.width, tid = threadIdx.x, nt = blockDim.x;
    for(int s = blockIdx.x; s < p.n_streams; s += gridDim.x)
    {
        float *r0 = ring, *r1 = ring + W;
        for(int i = tid; i < 2 * W; i += nt)
            ring[i] = p.state[(size_t)s * 2 * W + i];
        int head = 0;
        bool last_silent = p.flags[s] != 0;
        const float *pcm0 = p.pcm + (size_t)s * p.stream_stride;
        const float *pcm1 = pcm0 + p.channel_stride;
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
                r0[pos] = (q >= 0) ? __ldg(pcm0 + q) : 0.0f;
                if(p.cc > 1)
                    r1[pos] = (q >= 0) ? __ldg(pcm1 + q) : 0.0f;
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
            float *orow = p.out + ((size_t)s * p.n_ticks + t) * p.dch * W;
            for(int d = 0; d < p.dch; ++d)
                for(int i = tid; i < W; i += nt)
                {
                    int pos = head + i;
                    pos -= (pos >= W) ? W : 0;
                    __stcs(orow + d * W + i, ring[d * W + pos]);
                }
            if(p.out_silent != nullptr && tid == 0)
                p.out_silent[(size_t)s * p.n_ticks + t] = last_silent ? 1 : 0;
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

template<int MODE>
__global__ void __launch_bounds__(256, 5) wave_chunk_kernel(const WParams p)
{
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
        const float *pcm0 = p.pcm + (size_t)s * p.stream_stride;
        const float *pcm1 = pcm0 + p.channel_stride;
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
                        ra[u] = (q[u] >= 0) ? __ldg(pcm0 + q[u]) : 0.0f;
                        rb[u] = (TWO && q[u] >= 0) ? __ldg(pcm1 + q[u]) : 0.0f;
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
            // rows of ticks [t, t+Kc): windows of E in time order
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
                        __stcs(p.out + (((size_t)s * p.n_ticks + t + j) * DCH + d) * W + i, v);
                        if(wr_state1 && d == 1 && j == Kc - 1)
                            st1[i] = v;
                    }
                }
                if(p.out_silent != nullptr && tid < Kc)
                    p.out_silent[(size_t)s * p.n_ticks + t + tid] = (hit && tid == Kc - 1) ? 1 : 0;
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

__global__ void wave_fill_kernel(float *q, long long n, float v)
{
    for(long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        q[i] = v;
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

// util.hpp's audio_frames_to_ns / ns_to_audio_frames (128-bit multiply-divide).  The 64-bit form is the same quotient
// whenever the product fits, which it does for everything but multi-day spans; the 128-bit division costs ~50 ns and the
// plan evaluates one per point.
uint64_t frames_to_ns(uint64_t sr, uint64_t frames)
{
    if(frames <= UINT64_MAX / 1000000000ull)
        return (frames * 1000000000ull) / sr;
    return (uint64_t)(((unsigned __int128)frames * 1000000000ull) / sr);
}
uint64_t ns_to_frames(uint64_t sr, uint64_t ns)
{
    if(ns <= UINT64_MAX / sr)
        return (ns * sr) / 1000000000ull;
    return (uint64_t)(((unsigned __int128)ns * sr) / 1000000000ull);
}

} // namespace

struct wf_wave {
    wf_wave_config cfg{};
    int device = 0, sm_count = 0;
    int dch = 1, och = 1;
    size_t ws = 0;        // m_waveform_samples
    float db_min = 0.0f;
    // the clock the reference derives from packet timestamps (shared by all streams: they tick together)
    uint64_t clock = 10ull * 1000000000ull, audio_ts = 0, waveform_ts = 0;
    size_t prefill = 0;   // start-up zeros still pending in the capture ring (src/source.cpp:1243-1248)
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool ev_valid = false;
    std::string last_error;
    int64_t launches = 0;
    float *d_state = nullptr;
    unsigned char *d_flags = nullptr;
    int *d_src = nullptr, *d_off = nullptr;
    float *s_pcm = nullptr, *s_out = nullptr, *s_rms = nullptr;
    unsigned char *s_silent = nullptr;
    size_t src_cap = 0, off_cap = 0, pcm_cap = 0, out_cap = 0, rms_cap = 0, silent_cap = 0;
    struct PlanSlot {
        int *h = nullptr; // pinned: off[] then src[]
        size_t cap = 0;
        cudaEvent_t done = nullptr;
        bool used = false;
    };
    static constexpr int kSlots = 4;
    PlanSlot slots[kSlots];
    int slot_next = 0;
    cudaStream_t last_stream = nullptr;
    bool chunked = true;  // wave_chunk_kernel (WF_WAVE_CHUNK=0: the per-tick kernel, kept for A/B and bit-identity tests)
    int chunk_mode = 0, chunk_floats = 0, chunk_per_sm = 8;
};

namespace {

thread_local std::string g_wave_create_error;

int werr(wf_wave *w, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if(w)
        w->last_error = buf;
    else
        g_wave_create_error = buf;
    return code;
}

#define WFW_CUDA(w, call)                                                                                       \
    do                                                                                                          \
    {                                                                                                           \
        cudaError_t _err = (call);                                                                              \
        if(_err != cudaSuccess)                                                                                 \
            return werr((w), (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s failed: %s", \
                        #call, cudaGetErrorString(_err));                                                       \
    } while(0)

template<typename T>
int wensure(wf_wave *w, T **buf, size_t *cap, size_t need)
{
    if(need <= *cap)
        return WF_OK;
    if(*buf)
        cudaFree(*buf);
    *buf = nullptr;
    *cap = 0;
    WFW_CUDA(w, cudaMalloc((void **)buf, need * sizeof(T)));
    *cap = need;
    return WF_OK;
}

bool w_is_device_ptr(const void *p)
{
    if(!p)
        return false;
    cudaPointerAttributes a{};
    if(cudaPointerGetAttributes(&a, p) != cudaSuccess)
    {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// The tick-by-tick timestamp walk of tick_waveform (src/source_generic.cpp:303-339,358) for packets of `hop` samples that
// end "now": appends, per tick, the source sample of every new point (index into the call's PCM, -1 = start-up zero).
void plan_ticks(wf_wave *w, int n_ticks, int hop, std::vector<int> &src, std::vector<int> &off)
{
    const uint64_t sr = w->cfg.sample_rate;
    const size_t outsz = (size_t)w->cfg.width;
    const uint64_t step_ns = ((uint64_t)w->cfg.meter_ms * 1000000ull) / (uint64_t)outsz; // :303
    src.clear();
    off.assign(1, 0);
    for(int t = 0; t < n_ticks; ++t)
    {
        w->clock += frames_to_ns(sr, (uint64_t)hop);
        w->audio_ts = w->clock; // timestamp + audio_len, src/source.cpp:1836
        const size_t avail = w->prefill + (size_t)hop;
        const size_t total = std::min(avail, w->ws); // the ring keeps m_waveform_samples (src/source.cpp:1881-1884)
        const size_t skip = avail - total;
        const size_t prefill = w->prefill;
        w->prefill = 0;
        size_t count = 0;
        if(total > 0)
        {
            const uint64_t start_ts = w->audio_ts - frames_to_ns(sr, total), stop_ts = w->audio_ts;
            if(!((start_ts >= w->audio_ts) || (stop_ts > w->audio_ts))) // :321-322
            {
                if(w->waveform_ts < start_ts)
                    w->waveform_ts = start_ts; // :323-324
                if((w->waveform_ts > stop_ts) && ((w->waveform_ts - stop_ts) > step_ns))
                    w->waveform_ts = start_ts; // :325-326
                for(size_t i = 0; i < outsz; ++i)
                {
                    const uint64_t ts = w->waveform_ts + (i * step_ns);
                    if(ts >= stop_ts || ts < w->waveform_ts)
                        break;
                    const uint64_t index = std::clamp<uint64_t>(ns_to_frames(sr, w->audio_ts - ts), 1u, total); // :336
                    const size_t pos = skip + (total - index); // position in (start-up zeros ++ packet)
                    src.push_back(pos < prefill ? -1 : (int)((size_t)t * hop + (pos - prefill)));
                    ++count;
                }
                w->waveform_ts += count * step_ns; // :358
            }
        }
        off.push_back((int)src.size());
    }
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
}

const char *wf_wave_last_error(const wf_wave *w) { return w ? w->last_error.c_str() : g_wave_create_error.c_str(); }

int wf_wave_create(const wf_wave_config *cfg, wf_wave **out)
{
    if(!cfg || !out)
        return WF_ERR_INVALID_ARG;
    *out = nullptr;
    if(cfg->struct_size != sizeof(wf_wave_config))
        return werr(nullptr, WF_ERR_ABI, "wf_wave_config.struct_size mismatch");
    if(cfg->capture_channels < 1 || cfg->capture_channels > 2 || cfg->max_streams < 1 || cfg->sample_rate < 1 ||
       cfg->width < 1 || cfg->width > 8192 || cfg->meter_ms < 1)
        return werr(nullptr, WF_ERR_INVALID_ARG, "bad waveform config");
    if(((uint64_t)cfg->meter_ms * 1000000ull) / (uint64_t)cfg->width == 0)
        return werr(nullptr, WF_ERR_INVALID_ARG, "meter_ms too small for this width (step of 0 ns)");
    int ndev = 0;
    if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    {
        cudaGetLastError();
        return werr(nullptr, WF_ERR_NO_DEVICE, "no CUDA device (the waveform mode has no CPU fallback)");
    }
    int dev = cfg->device;
    if(dev < 0 && cudaGetDevice(&dev) != cudaSuccess)
        return werr(nullptr, WF_ERR_CUDA, "cudaGetDevice failed");
    if(dev >= ndev)
        return werr(nullptr, WF_ERR_INVALID_ARG, "device %d out of range", dev);
    wf_wave *w = new(std::nothrow) wf_wave();
    if(!w)
        return WF_ERR_OOM;
    w->cfg = *cfg;
    w->device = dev;
    w->dch = cfg->stereo ? 2 : 1;
    w->och = ((cfg->capture_channels > 1) || cfg->stereo) ? 2 : 1; // src/source.cpp:1171
    w->ws = (size_t)((double)cfg->sample_rate * ((double)cfg->meter_ms / 1000.0)); // :1141
    w->prefill = (size_t)cfg->width;                                               // :1243-1248 (m_fft_size zeros)
    w->db_min = 20.0f * log10f(1.17549435e-38f);
    auto bail = [&](int code) {
        g_wave_create_error = w->last_error;
        wf_wave_destroy(w);
        return code;
    };
#define WFW_C(call)                                                                                  \
    do                                                                                               \
    {                                                                                                \
        cudaError_t _err = (call);                                                                   \
        if(_err != cudaSuccess)                                                                      \
            return bail(werr(w, (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s: %s", #call, \
                             cudaGetErrorString(_err)));                                             \
    } while(0)
    WFW_C(cudaSetDevice(dev));
    cudaDeviceProp prop{};
    WFW_C(cudaGetDeviceProperties(&prop, dev));
    if(prop.major != 9 || prop.minor != 0) // sm_90a code runs on compute capability 9.0 only
        return bail(werr(w, WF_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major,
                         prop.minor));
    w->sm_count = prop.multiProcessorCount;
    if(2 * (size_t)cfg->width * sizeof(float) > 48 * 1024) // widths above 6144: both scrolling rings exceed the default 48 KB
        WFW_C(cudaFuncSetAttribute(wave_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(2 * (size_t)cfg->width * sizeof(float))));
    {
        const char *e = getenv("WF_WAVE_CHUNK");
        w->chunked = !(e && e[0] == '0');
        const bool two = cfg->capture_channels > 1;
        w->chunk_mode = cfg->stereo ? (two ? 2 : 3) : (two ? 1 : 0);
        static const int mult[4] = {2, 4, 4, 3};
        w->chunk_floats = mult[w->chunk_mode] * cfg->width;
        const int bytes = w->chunk_floats * (int)sizeof(float);
        if(bytes > 48 * 1024)
        {
            switch(w->chunk_mode)
            {
            case 0: WFW_C(cudaFuncSetAttribute(wave_chunk_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); break;
            case 1: WFW_C(cudaFuncSetAttribute(wave_chunk_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); break;
            case 2: WFW_C(cudaFuncSetAttribute(wave_chunk_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); break;
            default: WFW_C(cudaFuncSetAttribute(wave_chunk_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); break;
            }
        }
        int per_sm = 0;
        switch(w->chunk_mode)
        {
        case 0: WFW_C(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wave_chunk_kernel<0>, 256, (size_t)bytes)); break;
        case 1: WFW_C(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wave_chunk_kernel<1>, 256, (size_t)bytes)); break;
        case 2: WFW_C(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wave_chunk_kernel<2>, 256, (size_t)bytes)); break;
        default: WFW_C(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wave_chunk_kernel<3>, 256, (size_t)bytes)); break;
        }
        w->chunk_per_sm = std::max(1, per_sm); // one resident wave: streams are equal work, a partial second wave is a tail
    }
    WFW_C(cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking));
    WFW_C(cudaEventCreate(&w->ev0));
    WFW_C(cudaEventCreate(&w->ev1));
    const size_t S = (size_t)cfg->max_streams, n = S * 2 * (size_t)cfg->width;
    WFW_C(cudaMalloc((void **)&w->d_state, n * sizeof(float)));
    WFW_C(cudaMalloc((void **)&w->d_flags, S));
    WFW_C(cudaMemsetAsync(w->d_flags, 0, S, w->stream)); // m_last_silent := false, src/source.cpp:1236
    wave_fill_kernel<<<(int)std::min<size_t>((n + 255) / 256, 2048), 256, 0, w->stream>>>(w->d_state, (long long)n, w->db_min);
    WFW_C(cudaGetLastError());
    w->launches++;
    WFW_C(cudaStreamSynchronize(w->stream));
#undef WFW_C
    *out = w;
    return WF_OK;
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
    void *ptrs[] = {w->d_state, w->d_flags, w->d_src, w->d_off, w->s_pcm, w->s_out, w->s_rms, w->s_silent};
    for(void *q : ptrs)
        if(q)
            cudaFree(q);
    for(auto &ps : w->slots)
    {
        if(ps.h)
            cudaFreeHost(ps.h);
        if(ps.done)
            cudaEventDestroy(ps.done);
    }
    if(w->ev0)
        cudaEventDestroy(w->ev0);
    if(w->ev1)
        cudaEventDestroy(w->ev1);
    if(w->stream)
        cudaStreamDestroy(w->stream);
    delete w;
}

int wf_wave_process_async(wf_wave *w, const wf_wave_batch *b, void *cuda_stream)
{
    if(!w || !b)
        return WF_ERR_INVALID_ARG;
    wf::NvtxRange nvtx("wf_wave_process");
    if(b->struct_size != sizeof(wf_wave_batch))
        return werr(w, WF_ERR_ABI, "wf_wave_batch.struct_size %u != %zu", b->struct_size, sizeof(wf_wave_batch));
    if(b->n_ticks < 0 || b->hop < 1)
        return werr(w, WF_ERR_INVALID_ARG, "n_ticks must be >= 0 and hop >= 1");
    if(b->n_streams != w->cfg.max_streams)
        return werr(w, WF_ERR_CAPACITY, "a waveform call must tick all %d streams of the engine (got %d): the clock is shared",
                    w->cfg.max_streams, b->n_streams);
    if(b->n_ticks == 0)
        return WF_OK;
    if(!b->pcm || !b->out)
        return werr(w, WF_ERR_INVALID_ARG, "pcm / out is null");
    if(b->stream_stride < 0 || b->channel_stride < 0)
        return werr(w, WF_ERR_INVALID_ARG, "negative strides are not supported");
    if((long long)b->n_ticks * b->hop > 0x7fffffffLL)
        return werr(w, WF_ERR_INVALID_ARG, "n_ticks * hop too large for one call");

    WFW_CUDA(w, cudaSetDevice(w->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : w->stream;
    const int cc = w->cfg.capture_channels, W = w->cfg.width;
    const size_t S = (size_t)b->n_streams, T = (size_t)b->n_ticks;
    std::vector<int> src, off;
    plan_ticks(w, b->n_ticks, b->hop, src, off);
    int rc;
    if((rc = wensure(w, &w->d_src, &w->src_cap, std::max<size_t>(1, src.size()))))
        return rc;
    if((rc = wensure(w, &w->d_off, &w->off_cap, off.size())))
        return rc;
    {
        // the plan goes through one of a few pinned slots, so a call neither waits for the previous kernel nor leaves the
        // device reading a vector that is about to go away; a slot is reused only after its copy has completed
        wf_wave::PlanSlot &ps = w->slots[w->slot_next];
        w->slot_next = (w->slot_next + 1) % wf_wave::kSlots;
        if(ps.used)
            WFW_CUDA(w, cudaEventSynchronize(ps.done));
        const size_t need = src.size() + off.size();
        if(need > ps.cap)
        {
            if(ps.h)
                cudaFreeHost(ps.h);
            ps.h = nullptr;
            ps.cap = 0;
            WFW_CUDA(w, cudaMallocHost((void **)&ps.h, need * sizeof(int)));
            ps.cap = need;
        }
        if(!ps.done)
            WFW_CUDA(w, cudaEventCreateWithFlags(&ps.done, cudaEventDisableTiming));
        memcpy(ps.h, off.data(), off.size() * sizeof(int));
        if(!src.empty())
            memcpy(ps.h + off.size(), src.data(), src.size() * sizeof(int));
        if(w->last_stream != nullptr && w->last_stream != st)
            WFW_CUDA(w, cudaStreamSynchronize(w->last_stream)); // d_src / d_off may still be read by a call on another stream
        w->last_stream = st;
        WFW_CUDA(w, cudaMemcpyAsync(w->d_off, ps.h, off.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        if(!src.empty())
            WFW_CUDA(w, cudaMemcpyAsync(w->d_src, ps.h + off.size(), src.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WFW_CUDA(w, cudaEventRecord(ps.done, st));
        ps.used = true;
    }

    const bool dev_ptrs = w_is_device_ptr(b->pcm);
    const float *d_pcm = b->pcm, *d_rms = b->input_rms;
    float *d_out = b->out;
    unsigned char *d_silent = b->out_silent;
    const size_t out_n = S * T * w->dch * (size_t)W;
    if(!dev_ptrs)
    {
        const size_t span = (S - 1) * (size_t)b->stream_stride + (size_t)(cc - 1) * (size_t)b->channel_stride + T * (size_t)b->hop;
        if((rc = wensure(w, &w->s_pcm, &w->pcm_cap, span)))
            return rc;
        WFW_CUDA(w, cudaMemcpyAsync(w->s_pcm, b->pcm, span * sizeof(float), cudaMemcpyHostToDevice, st));
        d_pcm = w->s_pcm;
        if((rc = wensure(w, &w->s_out, &w->out_cap, out_n)))
            return rc;
        d_out = w->s_out;
        if(b->input_rms)
        {
            if((rc = wensure(w, &w->s_rms, &w->rms_cap, S * T)))
                return rc;
            WFW_CUDA(w, cudaMemcpyAsync(w->s_rms, b->input_rms, S * T * sizeof(float), cudaMemcpyHostToDevice, st));
            d_rms = w->s_rms;
        }
        if(b->out_silent)
        {
            if((rc = wensure(w, &w->s_silent, &w->silent_cap, S * T)))
                return rc;
            d_silent = w->s_silent;
        }
    }
    WParams p{};
    p.pcm = d_pcm;
    p.stream_stride = b->stream_stride;
    p.channel_stride = b->channel_stride;
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
    WFW_CUDA(w, cudaEventRecord(w->ev0, st));
    const int grid = (int)std::min<size_t>(S, (size_t)w->sm_count * (w->chunked ? w->chunk_per_sm : 8));
    if(w->chunked)
    {
        const size_t smem = (size_t)w->chunk_floats * sizeof(float);
        switch(w->chunk_mode)
        {
        case 0: wave_chunk_kernel<0><<<grid, 256, smem, st>>>(p); break;
        case 1: wave_chunk_kernel<1><<<grid, 256, smem, st>>>(p); break;
        case 2: wave_chunk_kernel<2><<<grid, 256, smem, st>>>(p); break;
        default: wave_chunk_kernel<3><<<grid, 256, smem, st>>>(p); break;
        }
    }
    else
        wave_kernel<<<grid, 256, 2 * (size_t)W * sizeof(float), st>>>(p);
    WFW_CUDA(w, cudaGetLastError());
    w->launches++;
    WFW_CUDA(w, cudaEventRecord(w->ev1, st));
    w->ev_valid = true;
    if(!dev_ptrs)
    {
        WFW_CUDA(w, cudaMemcpyAsync(b->out, d_out, out_n * sizeof(float), cudaMemcpyDeviceToHost, st));
        if(b->out_silent)
            WFW_CUDA(w, cudaMemcpyAsync(b->out_silent, d_silent, S * T, cudaMemcpyDeviceToHost, st));
    }
    return WF_OK;
}

int wf_wave_process(wf_wave *w, const wf_wave_batch *b)
{
    int rc = wf_wave_process_async(w, b, nullptr);
    if(rc)
        return rc;
    WFW_CUDA(w, cudaStreamSynchronize(w->stream));
    return WF_OK;
}

int wf_wave_reset(wf_wave *w)
{
    if(!w)
        return WF_ERR_INVALID_ARG;
    WFW_CUDA(w, cudaSetDevice(w->device));
    wave_reset_kernel<<<std::min(w->cfg.max_streams, w->sm_count * 4), 256, 0, w->stream>>>(w->d_state, w->d_flags,
                                                                                          w->cfg.max_streams, w->dch,
                                                                                          w->cfg.width, w->db_min);
    WFW_CUDA(w, cudaGetLastError());
    w->launches++;
    WFW_CUDA(w, cudaStreamSynchronize(w->stream));
    return WF_OK;
}

int64_t wf_wave_preview_plan(const wf_wave_config *cfg, int32_t n_ticks, int32_t hop, int32_t *counts, int32_t *src,
                             int64_t capacity)
{
    if(!cfg || n_ticks < 0 || hop < 1)
        return WF_ERR_INVALID_ARG;
    if(cfg->struct_size != sizeof(wf_wave_config))
        return WF_ERR_ABI;
    if(cfg->sample_rate < 1 || cfg->width < 1 || cfg->width > 8192 || cfg->meter_ms < 1 ||
       ((uint64_t)cfg->meter_ms * 1000000ull) / (uint64_t)cfg->width == 0)
        return WF_ERR_INVALID_ARG;
    wf_wave w; // host-only use: the same initial clock / start-up state wf_wave_create sets up
    w.cfg = *cfg;
    w.ws = (size_t)((double)cfg->sample_rate * ((double)cfg->meter_ms / 1000.0));
    w.prefill = (size_t)cfg->width;
    std::vector<int> s, off;
    plan_ticks(&w, n_ticks, hop, s, off);
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

int64_t wf_wave_launch_count(const wf_wave *w) { return w ? w->launches : 0; }

float wf_wave_last_kernel_ms(wf_wave *w)
{
    if(!w || !w->ev_valid || cudaEventSynchronize(w->ev1) != cudaSuccess)
        return -1.0f;
    float ms = -1.0f;
    if(cudaEventElapsedTime(&ms, w->ev0, w->ev1) != cudaSuccess)
        return -1.0f;
    return ms;
}

} // extern "C"
