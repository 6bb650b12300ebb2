// wf_meter.cu — level meter (tick_meter) and RMS feed (update_input_rms) of the plugin as batched sm_90a reductions
// behind the C ABI of include/wfstft.h (wf_meter_*).  SURVEY.md §8(f) rank 4 / §8(a) row a9.
//
// Reference semantics restated (paths relative to the reference tree):
//   tick_meter          src/source_generic.cpp:182-270: ring of the last W samples -> RMS or peak -> EMA -> dBFS -> silent
//   update_input_rms    src/source_generic.cpp:392-403 + src/source.cpp:810-836,1842-1871: ring of the last RW values
//                       (max over channels |x|)^2 -> sqrt(mean)
//
// HBM-bound integer/float streaming work, so the design is about touching each sample once:
//   K1 block partials   every block of the stream's timeline (history ring ++ new PCM) is reduced once (sum of squares /
//                       max |x| / sum of (max_c |x_c|)^2) with 128-bit loads; the block size is the largest power of two
//                       (32..256) dividing hop and W, so that windows are whole numbers of blocks whenever possible;
//   K2 window combine   one warp per (stream, tick, channel): whole blocks from the partials (L2-resident) + ragged
//                       edges from the samples if any — O(W/block) instead of O(W) per tick, windows overlap W/hop times;
//   K3 recurrence       one thread per stream walks the ticks: sqrt/mean, EMA (fast-peaks rule), dBFS, m_last_silent;
//   (history)           K1 also writes the last W samples of the timeline into the (double-buffered) ring for the next call.
// There is no CPU fallback.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "wf_nvtx.hpp"
#include "wf_tables.hpp"
#include "wfstft.h"

namespace {

constexpr int kChunk = 256; // samples one warp reduces in K1 (8 per lane); partial blocks are 32..256 samples

struct MParams {
    const float *pcm;
    long long stream_stride, channel_stride;
    const float *hist;   // [streams][cc][W] time-ordered ring contents before this call
    float *hist_next;    // same layout, after this call
    float *partial;      // [streams][pc][nblk]
    const float *part_in; // one-pass path: the W/hop block partials of the ring as the previous call left them, or null (reduce the ring)
    float *part_out;      // one-pass path: this call's last W/hop block partials [streams][pc][W/hop]
    float *raw;          // [streams][ticks][pc]
    float *buf;          // [streams][2] m_meter_buf
    unsigned char *flags;// [streams] m_last_silent
    float *out_db, *out_lin;
    unsigned char *out_silent;
    int n_streams, n_ticks, hop, W, cc, pc, nblk, mode;
    int bl;    // samples per partial: the largest power of two <= 256 dividing both hop and W (then windows have no ragged edges), else 256
    int nchunk;// 256-sample chunks of the timeline (one warp each in K1)
    float g, g2;
    int tsmooth, fast_peaks;
    float floor_m10, db_min;
};

// Row pointers of one (stream, channel): history ring first (timeline positions [0, W)), then this call's PCM.
struct Row {
    const float *hist, *pcm;
};
__device__ __forceinline__ Row row_of(const MParams &p, int s, int c)
{
    return {p.hist + ((size_t)s * p.cc + c) * p.W, p.pcm + (size_t)s * p.stream_stride + (size_t)c * p.channel_stride};
}
__device__ __forceinline__ float vsample(const Row &r, int W, long long u)
{
    return (u < W) ? r.hist[u] : __ldg(r.pcm + (u - W));
}

template<int MODE>
__device__ __forceinline__ float combine(float a, float b)
{
    return (MODE == WF_METER_PEAK) ? fmaxf(a, b) : __fadd_rn(a, b);
}
// what one sample contributes: x^2 (RMS), |x| (peak), (max over channels |x|)^2 (RMS feed, src/source.cpp:1852-1862)
template<int MODE>
__device__ __forceinline__ float contrib(float x0, float x1)
{
    if(MODE == WF_METER_INPUT_RMS)
    {
        const float v = fmaxf(fabsf(x1), fmaxf(fabsf(x0), 0.0f));
        return __fmul_rn(v, v);
    }
    return (MODE == WF_METER_RMS) ? __fmul_rn(x0, x0) : fabsf(x0);
}
template<int MODE>
__device__ __forceinline__ float warp_combine(float v)
{
#pragma unroll
    for(int o = 16; o > 0; o >>= 1)
        v = combine<MODE>(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// scalar reduction of timeline positions [lo, hi) by one warp (ragged edges, history, unaligned PCM)
template<int MODE>
__device__ __forceinline__ float reduce_range(const Row &r0, const Row &r1, bool two, int W, long long lo, long long hi,
                                              int lane, float acc)
{
    for(long long u = lo + lane; u < hi; u += 32)
    {
        const float x0 = vsample(r0, W, u);
        const float x1 = (MODE == WF_METER_INPUT_RMS && two) ? vsample(r1, W, u) : 0.0f;
        acc = combine<MODE>(acc, contrib<MODE>(x0, x1));
    }
    return acc;
}

// K1: one warp per (stream, partial channel, 256-sample chunk): lane l reduces samples [8l, 8l+8) of the chunk, groups of
// bl/8 lanes combine into one partial per bl-sample block.  Chunks that lie wholly inside 16-byte aligned new PCM (all
// but the few that touch the history ring or the end) take two 128-bit loads per lane.  The same pass writes the last W
// samples of the timeline into the ring for the next call (every sample is read exactly once here).
template<int MODE>
__global__ void meter_block_kernel(const MParams p, const int vec4)
{
    const int warps_per_cta = blockDim.x >> 5;
    const int lane = threadIdx.x & 31;
    const long long total = (long long)p.n_streams * p.pc * p.nchunk;
    const long long L = (long long)p.W + (long long)p.n_ticks * p.hop;
    const long long tail0 = L - p.W; // timeline position of ring slot 0 of the next call
    const bool two = (MODE == WF_METER_INPUT_RMS) && p.cc > 1;
    const int per = kChunk / p.bl;   // partials per chunk
    const int glanes = p.bl / 8;     // lanes per partial
    for(long long w = (long long)blockIdx.x * warps_per_cta + (threadIdx.x >> 5); w < total;
        w += (long long)gridDim.x * warps_per_cta)
    {
        const int j = (int)(w % p.nchunk);
        const int c = (int)((w / p.nchunk) % p.pc);
        const int s = (int)(w / ((long long)p.nchunk * p.pc));
        const long long u0 = (long long)j * kChunk;
        const Row r0 = row_of(p, s, c);
        const Row r1 = two ? row_of(p, s, 1) : r0;
        float *h0 = p.hist_next + ((size_t)s * p.cc + c) * p.W;
        float *h1 = p.hist_next + ((size_t)s * p.cc + 1) * p.W;
        float acc = 0.0f;
        const long long ul = u0 + 8 * lane; // my 8 samples
        if(vec4 && u0 >= p.W && u0 + kChunk <= L)
        {
            const float4 *q0 = reinterpret_cast<const float4 *>(r0.pcm + (ul - p.W));
            const float4 a = __ldg(q0), b = __ldg(q0 + 1);
            float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = a1;
            if(two)
            {
                const float4 *q1 = reinterpret_cast<const float4 *>(r1.pcm + (ul - p.W));
                a1 = __ldg(q1);
                b1 = __ldg(q1 + 1);
            }
            acc = combine<MODE>(combine<MODE>(contrib<MODE>(a.x, a1.x), contrib<MODE>(a.y, a1.y)),
                                combine<MODE>(contrib<MODE>(a.z, a1.z), contrib<MODE>(a.w, a1.w)));
            acc = combine<MODE>(acc, combine<MODE>(combine<MODE>(contrib<MODE>(b.x, b1.x), contrib<MODE>(b.y, b1.y)),
                                                   combine<MODE>(contrib<MODE>(b.z, b1.z), contrib<MODE>(b.w, b1.w))));
            if(ul + 8 > tail0)
            {
                // ring for the next call (tail0 is a multiple of 4 here: W, n_ticks*hop offsets keep 16-byte alignment
                // only if hop is a multiple of 4 -> otherwise fall back to scalar stores)
                if(ul >= tail0 && ((tail0 & 3) == 0))
                {
                    *reinterpret_cast<float4 *>(h0 + (ul - tail0)) = a;
                    *reinterpret_cast<float4 *>(h0 + (ul - tail0) + 4) = b;
                    if(two)
                    {
                        *reinterpret_cast<float4 *>(h1 + (ul - tail0)) = a1;
                        *reinterpret_cast<float4 *>(h1 + (ul - tail0) + 4) = b1;
                    }
                }
                else
                {
                    const float va[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                    const float vb[8] = {a1.x, a1.y, a1.z, a1.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                    for(int i = 0; i < 8; ++i)
                        if(ul + i >= tail0)
                        {
                            h0[ul + i - tail0] = va[i];
                            if(two)
                                h1[ul + i - tail0] = vb[i];
                        }
                }
            }
        }
        else
        {
#pragma unroll
            for(int i = 0; i < 8; ++i)
            {
                const long long u = ul + i;
                if(u < L)
                {
                    const float x0 = vsample(r0, p.W, u);
                    const float x1 = two ? vsample(r1, p.W, u) : 0.0f;
                    acc = combine<MODE>(acc, contrib<MODE>(x0, x1));
                    if(u >= tail0)
                    {
                        h0[u - tail0] = x0;
                        if(two)
                            h1[u - tail0] = x1;
                    }
                }
            }
        }
        // combine inside each group of glanes lanes (= one partial of bl samples)
        for(int o = 1; o < glanes; o <<= 1)
            acc = combine<MODE>(acc, __shfl_xor_sync(0xffffffffu, acc, o));
        if((lane & (glanes - 1)) == 0)
        {
            const long long blk = (long long)j * per + lane / glanes;
            if(blk < p.nblk)
                p.partial[((size_t)s * p.pc + c) * p.nblk + blk] = acc;
        }
    }
}

// K2: one warp per (stream, tick, partial channel): window [lo, hi) of the timeline
template<int MODE>
__global__ void meter_window_kernel(const MParams p)
{
    const int warps_per_cta = blockDim.x >> 5;
    const int lane = threadIdx.x & 31;
    const long long total = (long long)p.n_streams * p.n_ticks * p.pc;
    const bool two = (MODE == WF_METER_INPUT_RMS) && p.cc > 1;
    for(long long w = (long long)blockIdx.x * warps_per_cta + (threadIdx.x >> 5); w < total;
        w += (long long)gridDim.x * warps_per_cta)
    {
        const int c = (int)(w % p.pc);
        const int t = (int)((w / p.pc) % p.n_ticks);
        const int s = (int)(w / ((long long)p.pc * p.n_ticks));
        const long long lo = (long long)(t + 1) * p.hop, hi = lo + p.W;
        const long long jb = (lo + p.bl - 1) / p.bl, je = hi / p.bl;
        const Row r0 = row_of(p, s, c);
        const Row r1 = two ? row_of(p, s, 1) : r0;
        float acc = 0.0f;
        if(jb <= je)
        {
            acc = reduce_range<MODE>(r0, r1, two, p.W, lo, jb * p.bl, lane, acc);
            const float *part = p.partial + ((size_t)s * p.pc + c) * p.nblk;
            for(long long j = jb + lane; j < je; j += 32)
                acc = combine<MODE>(acc, part[j]);
            acc = reduce_range<MODE>(r0, r1, two, p.W, je * p.bl, hi, lane, acc);
        }
        else
            acc = reduce_range<MODE>(r0, r1, two, p.W, lo, hi, lane, acc);
        acc = warp_combine<MODE>(acc);
        if(lane == 0)
            p.raw[w] = acc;
    }
}

// K3: one thread per stream, the per-tick recurrence (src/source_generic.cpp:232-269)
__global__ void meter_scan_kernel(const MParams p)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if(s >= p.n_streams)
        return;
    if(p.mode == WF_METER_INPUT_RMS)
    {
        for(int t = 0; t < p.n_ticks; ++t)
            if(p.out_lin)
                p.out_lin[(size_t)s * p.n_ticks + t] =
                    __fsqrt_rn(__fdiv_rn(p.raw[(size_t)s * p.n_ticks + t], (float)p.W)); // src/source_generic.cpp:402
        return;
    }
    float buf[2] = {p.buf[2 * s], p.buf[2 * s + 1]};
    bool last_silent = p.flags[s] != 0;
    for(int t = 0; t < p.n_ticks; ++t)
    {
        int silent_channels = 0;
        for(int c = 0; c < p.cc; ++c)
        {
            float out = p.raw[((size_t)s * p.n_ticks + t) * p.pc + c];
            if(p.mode == WF_METER_RMS)
                out = __fsqrt_rn(__fdiv_rn(out, (float)p.W)); // :243
            if(p.tsmooth)
            {
                if(!p.fast_peaks || (out <= buf[c]))
                    out = __fadd_rn(__fmul_rn(p.g, buf[c]), __fmul_rn(p.g2, out)); // :255-256
            }
            buf[c] = out;
            const float val = (out > 0.0f) ? 20.0f * log10f(out) : p.db_min; // dbfs, src/source.hpp:293-299
            if(val < p.floor_m10)
                ++silent_channels;
            const size_t o = ((size_t)s * p.n_ticks + t) * p.cc + c;
            if(p.out_db)
                p.out_db[o] = val;
            if(p.out_lin)
                p.out_lin[o] = out;
        }
        last_silent = silent_channels >= p.cc; // :264-269
        if(p.out_silent)
            p.out_silent[(size_t)s * p.n_ticks + t] = last_silent ? 1 : 0;
    }
    p.buf[2 * s] = buf[0];
    p.buf[2 * s + 1] = buf[1];
    p.flags[s] = last_silent ? 1 : 0;
}

// ---- one-pass path: hop divides the window (the plugin's usual case: 150 ms at 48 kHz = 7200 = 9 x 800 samples at 60 fps) ----
// One CTA per stream.  Every hop-sized block of the stream's timeline (W/hop blocks of history ring, then one block per
// tick) is reduced ONCE by one warp with 128-bit loads — the same pass copies the last W samples into the next call's ring —
// and its partial lands in shared memory; a tick's window is then exactly W/hop consecutive partials, combined by one
// thread per (tick, channel); finally the per-stream recurrence (EMA, dBFS, m_last_silent) runs on one lane per channel.
// Samples cross HBM once, nothing else does: the three-kernel path above wrote and re-read per-32-sample partials W/hop times.
template<int MODE>
__global__ void __launch_bounds__(256) meter_fused_kernel(const MParams p)
{
    extern __shared__ float sm[];
    const int T = p.n_ticks, hop = p.hop, W = p.W, pc = p.pc, cc = p.cc;
    const int nb = W / hop, NB = nb + T;
    float *part = sm;                 // [pc][NB]
    float *raw = sm + (size_t)pc * NB; // [T][pc]
    const int s = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const bool two = (MODE == WF_METER_INPUT_RMS) && cc > 1;
    const int q4 = hop >> 2;
    // history blocks whose partials the previous call left behind (same hop): no need to read the ring again, unless the block
    // stays in the window beyond this call (T < W/hop) and therefore has to be copied into the next ring
    const bool have_part = p.part_in != nullptr;
    if(have_part)
        for(int i = threadIdx.x; i < pc * nb; i += blockDim.x)
            part[(i / nb) * NB + (i % nb)] = p.part_in[(size_t)s * pc * nb + i];
    for(int w = warp; w < pc * NB; w += nwarps)
    {
        const int c = w / NB, b = w - c * NB;
        if(have_part && b < nb && b < T)
            continue;
        const Row r0 = row_of(p, s, c);
        const Row r1 = two ? row_of(p, s, 1) : r0;
        const float4 *src0 = reinterpret_cast<const float4 *>((b < nb) ? r0.hist + (size_t)b * hop : r0.pcm + (size_t)(b - nb) * hop);
        const float4 *src1 = reinterpret_cast<const float4 *>((b < nb) ? r1.hist + (size_t)b * hop : r1.pcm + (size_t)(b - nb) * hop);
        const bool keep = b >= T; // one of the last W/hop blocks: belongs to the next call's ring
        float4 *h0 = reinterpret_cast<float4 *>(p.hist_next + ((size_t)s * cc + c) * W + (size_t)(b - T) * hop);
        float4 *h1 = reinterpret_cast<float4 *>(p.hist_next + ((size_t)s * cc + 1) * W + (size_t)(b - T) * hop);
        float acc = 0.0f;
        // four 128-bit loads in flight per lane and channel (a hop of 800 samples is 6.25 loads per lane)
        for(int i0 = lane; i0 < q4; i0 += 128)
        {
            float4 a[4], a1[4];
#pragma unroll
            for(int u = 0; u < 4; ++u)
            {
                const int i = i0 + 32 * u;
                a[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                a1[u] = a[u];
                if(i < q4)
                {
                    a[u] = (b < nb) ? src0[i] : __ldg(src0 + i);
                    if(two)
                        a1[u] = (b < nb) ? src1[i] : __ldg(src1 + i);
                }
            }
#pragma unroll
            for(int u = 0; u < 4; ++u)
            {
                const int i = i0 + 32 * u;
                if(i < q4) // (zeros would be neutral for all three modes, but the ring must only take real samples)
                {
                    acc = combine<MODE>(acc, combine<MODE>(combine<MODE>(contrib<MODE>(a[u].x, a1[u].x), contrib<MODE>(a[u].y, a1[u].y)),
                                                           combine<MODE>(contrib<MODE>(a[u].z, a1[u].z), contrib<MODE>(a[u].w, a1[u].w))));
                    if(keep)
                    {
                        h0[i] = a[u];
                        if(two)
                            h1[i] = a1[u];
                    }
                }
            }
        }
        acc = warp_combine<MODE>(acc);
        if(lane == 0 && !(have_part && b < nb))
            part[c * NB + b] = acc;
    }
    __syncthreads();
    for(int i = threadIdx.x; i < pc * nb; i += blockDim.x) // the ring's partials for the next call
        p.part_out[(size_t)s * pc * nb + i] = part[(i / nb) * NB + T + (i % nb)];
    // window of tick t = blocks [t+1, t+1+nb); the RMS of the window (:243) is per tick, so it is taken here, in parallel
    for(int idx = threadIdx.x; idx < T * pc; idx += blockDim.x)
    {
        const int t = idx / pc, c = idx - t * pc;
        const float *q = part + c * NB + t + 1;
        float acc = q[0];
        for(int i = 1; i < nb; ++i)
            acc = combine<MODE>(acc, q[i]);
        if(MODE == WF_METER_RMS)
            acc = __fsqrt_rn(__fdiv_rn(acc, (float)W)); // :243
        raw[idx] = acc;
    }
    __syncthreads();
    if(MODE == WF_METER_INPUT_RMS)
    {
        for(int t = threadIdx.x; t < T; t += blockDim.x)
            if(p.out_lin)
                p.out_lin[(size_t)s * T + t] = __fsqrt_rn(__fdiv_rn(raw[t], (float)W)); // src/source_generic.cpp:402
        return;
    }
    // per-stream recurrence (src/source_generic.cpp:232-269).  Only the temporal smoothing is sequential (two dependent
    // operations per tick): lane c < cc of warp 0 walks its channel and leaves the smoothed value in place; dBFS, the silent
    // rule and the stores are per tick again and run on all threads.  (A CTA stays resident until its slowest warp is done:
    // with the whole tail on one lane — sqrt, divide, log10f and a ballot per tick — 30 % of a CTA's life had 7 of 8 warps idle.)
    if(warp == 0 && lane < cc)
    {
        const int c = lane;
        float buf = p.buf[2 * s + c];
        if(p.tsmooth)
        {
            for(int t = 0; t < T; ++t)
            {
                float out = raw[t * pc + c];
                if(!p.fast_peaks || (out <= buf))
                    out = __fadd_rn(__fmul_rn(p.g, buf), __fmul_rn(p.g2, out)); // :255-256
                buf = out;
                raw[t * pc + c] = out;
            }
        }
        else
            buf = raw[(T - 1) * pc + c];
        p.buf[2 * s + c] = buf;
    }
    __syncthreads();
    for(int t = threadIdx.x; t < T; t += blockDim.x)
    {
        int below = 0;
        for(int c = 0; c < cc; ++c)
        {
            const float out = raw[t * pc + c];
            const float val = (out > 0.0f) ? 20.0f * log10f(out) : p.db_min; // dbfs, src/source.hpp:293-299
            below += (val < p.floor_m10) ? 1 : 0;
            const size_t o = ((size_t)s * T + t) * cc + c;
            if(p.out_db)
                p.out_db[o] = val;
            if(p.out_lin)
                p.out_lin[o] = out;
        }
        const bool silent = below >= cc; // :264-269
        if(p.out_silent)
            p.out_silent[(size_t)s * T + t] = silent ? 1 : 0;
        if(t == T - 1)
            p.flags[s] = silent ? 1 : 0;
    }
}

__global__ void meter_fill_kernel(float *q, long long n, float v)
{
    for(long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        q[i] = v;
}

// timeout branch (src/source_generic.cpp:184-199) for streams [first, first+count)
__global__ void meter_reset_kernel(float *hist, float *buf, unsigned char *flags, int first, int count, int cc, int W)
{
    for(int s = first + blockIdx.x; s < first + count; s += gridDim.x)
    {
        if(flags[s] != 0)
            continue; // already silent: tick returns early
        for(long long i = threadIdx.x; i < (long long)cc * W; i += blockDim.x)
            hist[(size_t)s * cc * W + i] = 0.0f;
        __syncthreads();
        if(threadIdx.x == 0)
        {
            buf[2 * s] = 0.0f;
            buf[2 * s + 1] = 0.0f;
            flags[s] = 1;
        }
    }
}

} // namespace

struct wf_meter {
    wf_meter_config cfg{};
    int device = 0, sm_count = 0;
    int W = 0, pc = 1;
    float db_min = 0.0f;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool ev_valid = false;
    std::string last_error;
    int64_t launches = 0;
    float *d_hist[2] = {nullptr, nullptr};
    int cur = 0;
    // one-pass path: block partials of the ring, double-buffered like the ring; valid for `part_hop` (0 = not valid: reduce the ring)
    float *d_part[2] = {nullptr, nullptr};
    size_t part_cap = 0;
    int part_hop = 0, part_cur = 0;
    bool use_fused = true; // WF_METER_FUSED=0: always the three-kernel path (A/B tests)
    float *d_buf = nullptr;
    unsigned char *d_flags = nullptr;
    // scratch / staging
    float *d_partial = nullptr, *d_raw = nullptr, *s_pcm = nullptr, *s_db = nullptr, *s_lin = nullptr;
    unsigned char *s_silent = nullptr;
    size_t partial_cap = 0, raw_cap = 0, pcm_cap = 0, db_cap = 0, lin_cap = 0, silent_cap = 0;
};

namespace {

thread_local std::string g_meter_create_error;

int merr(wf_meter *m, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if(m)
        m->last_error = buf;
    else
        g_meter_create_error = buf;
    return code;
}

#define WFM_CUDA(m, call)                                                                                       \
    do                                                                                                          \
    {                                                                                                           \
        cudaError_t _err = (call);                                                                              \
        if(_err != cudaSuccess)                                                                                 \
            return merr((m), (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s failed: %s", \
                        #call, cudaGetErrorString(_err));                                                       \
    } while(0)

template<typename T>
int mensure(wf_meter *m, T **buf, size_t *cap, size_t need)
{
    if(need <= *cap)
        return WF_OK;
    if(*buf)
        cudaFree(*buf);
    *buf = nullptr;
    *cap = 0;
    WFM_CUDA(m, cudaMalloc((void **)buf, need * sizeof(T)));
    *cap = need;
    return WF_OK;
}

bool m_is_device_ptr(const void *p)
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

int grid_for(long long warps, int warps_per_cta, int sm_count)
{
    const long long ctas = (warps + warps_per_cta - 1) / warps_per_cta;
    return (int)std::max<long long>(1, std::min<long long>(ctas, (long long)sm_count * 16));
}

} // namespace

extern "C" {

void wf_meter_config_init(wf_meter_config *c)
{
    memset(c, 0, sizeof(*c));
    c->struct_size = (uint32_t)sizeof(wf_meter_config);
    c->device = -1;
    c->max_streams = 1;
    c->sample_rate = 48000;
    c->capture_channels = 2;
    c->mode = WF_METER_RMS; // P_RMS_MODE default true, src/source.cpp:167
    c->meter_ms = 150;      // P_METER_BUF default, src/source.cpp:166
    c->tsmoothing = WF_TSMOOTH_EXPONENTIAL;
    c->gravity = 0.65f;
    c->fast_peaks = 0;
    c->floor_db = -65;
}

const char *wf_meter_last_error(const wf_meter *m) { return m ? m->last_error.c_str() : g_meter_create_error.c_str(); }

int wf_meter_create(const wf_meter_config *cfg, wf_meter **out)
{
    if(!cfg || !out)
        return WF_ERR_INVALID_ARG;
    *out = nullptr;
    if(cfg->struct_size != sizeof(wf_meter_config))
        return merr(nullptr, WF_ERR_ABI, "wf_meter_config.struct_size mismatch");
    if(cfg->capture_channels < 1 || cfg->capture_channels > 2 || cfg->max_streams < 1 || cfg->sample_rate < 16 ||
       cfg->mode < WF_METER_PEAK || cfg->mode > WF_METER_INPUT_RMS)
        return merr(nullptr, WF_ERR_INVALID_ARG, "bad meter config");
    int W;
    if(cfg->mode == WF_METER_INPUT_RMS)
        W = (int)(cfg->sample_rate & ~15u); // m_input_rms_size, src/source.cpp:1148
    else
        W = (int)(((size_t)((double)cfg->sample_rate * ((double)cfg->meter_ms / 1000.0))) & ~(size_t)15); // :1121
    if(W < 16)
        return merr(nullptr, WF_ERR_INVALID_ARG, "meter window of %d ms is shorter than 16 samples", cfg->meter_ms);
    int ndev = 0;
    if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    {
        cudaGetLastError();
        return merr(nullptr, WF_ERR_NO_DEVICE, "no CUDA device (the meter has no CPU fallback)");
    }
    int dev = cfg->device;
    if(dev < 0 && cudaGetDevice(&dev) != cudaSuccess)
        return merr(nullptr, WF_ERR_CUDA, "cudaGetDevice failed");
    if(dev >= ndev)
        return merr(nullptr, WF_ERR_INVALID_ARG, "device %d out of range", dev);
    wf_meter *m = new(std::nothrow) wf_meter();
    if(!m)
        return WF_ERR_OOM;
    m->cfg = *cfg;
    m->device = dev;
    m->W = W;
    m->pc = (cfg->mode == WF_METER_INPUT_RMS) ? 1 : cfg->capture_channels;
    m->db_min = 20.0f * log10f(1.17549435e-38f); // DB_MIN, src/source.cpp:43
    auto bail = [&](int code) {
        g_meter_create_error = m->last_error;
        wf_meter_destroy(m);
        return code;
    };
#define WFM_C(call)                                                                                  \
    do                                                                                               \
    {                                                                                                \
        cudaError_t _err = (call);                                                                   \
        if(_err != cudaSuccess)                                                                      \
            return bail(merr(m, (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s: %s", #call, \
                             cudaGetErrorString(_err)));                                             \
    } while(0)
    {
        const char *mf = getenv("WF_METER_FUSED");
        m->use_fused = !(mf && mf[0] == '0');
    }
    WFM_C(cudaSetDevice(dev));
    cudaDeviceProp prop{};
    WFM_C(cudaGetDeviceProperties(&prop, dev));
    if(prop.major != 9 || prop.minor != 0) // sm_90a code runs on compute capability 9.0 only
        return bail(merr(m, WF_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev,
                         prop.major, prop.minor));
    m->sm_count = prop.multiProcessorCount;
    WFM_C(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    WFM_C(cudaEventCreate(&m->ev0));
    WFM_C(cudaEventCreate(&m->ev1));
    const size_t S = (size_t)cfg->max_streams, hist_n = S * cfg->capture_channels * (size_t)W;
    WFM_C(cudaMalloc((void **)&m->d_hist[0], hist_n * sizeof(float)));
    WFM_C(cudaMalloc((void **)&m->d_hist[1], hist_n * sizeof(float)));
    WFM_C(cudaMalloc((void **)&m->d_buf, S * 2 * sizeof(float)));
    WFM_C(cudaMalloc((void **)&m->d_flags, S));
    // ≙ update(): ring := 0 (src/source.cpp:1181), m_meter_buf := DB_MIN (:1124-1125, sic), m_last_silent := false (:1236)
    WFM_C(cudaMemsetAsync(m->d_hist[0], 0, hist_n * sizeof(float), m->stream));
    WFM_C(cudaMemsetAsync(m->d_flags, 0, S, m->stream));
    meter_fill_kernel<<<(int)std::min<size_t>((S * 2 + 255) / 256, 1024), 256, 0, m->stream>>>(m->d_buf, (long long)S * 2,
                                                                                              m->db_min);
    WFM_C(cudaGetLastError());
    m->launches++;
    WFM_C(cudaStreamSynchronize(m->stream));
#undef WFM_C
    *out = m;
    return WF_OK;
}

void wf_meter_destroy(wf_meter *m)
{
    if(!m)
        return;
    if(m->stream)
    {
        cudaSetDevice(m->device);
        cudaStreamSynchronize(m->stream);
    }
    void *ptrs[] = {m->d_part[0], m->d_part[1], m->d_hist[0], m->d_hist[1], m->d_buf, m->d_flags, m->d_partial, m->d_raw,
                    m->s_pcm, m->s_db, m->s_lin, m->s_silent};
    for(void *q : ptrs)
        if(q)
            cudaFree(q);
    if(m->ev0)
        cudaEventDestroy(m->ev0);
    if(m->ev1)
        cudaEventDestroy(m->ev1);
    if(m->stream)
        cudaStreamDestroy(m->stream);
    delete m;
}

int32_t wf_meter_window(const wf_meter *m) { return m ? m->W : 0; }

int wf_meter_process_async(wf_meter *m, const wf_meter_batch *b, void *cuda_stream)
{
    if(!m || !b)
        return WF_ERR_INVALID_ARG;
    wf::NvtxRange nvtx("wf_meter_process");
    if(b->struct_size != sizeof(wf_meter_batch))
        return merr(m, WF_ERR_ABI, "wf_meter_batch.struct_size %u != %zu", b->struct_size, sizeof(wf_meter_batch));
    if(b->n_streams < 0 || b->n_ticks < 0 || b->hop < 1)
        return merr(m, WF_ERR_INVALID_ARG, "n_streams/n_ticks must be >= 0 and hop >= 1");
    if(b->first_stream < 0 || (int64_t)b->first_stream + b->n_streams > m->cfg.max_streams)
        return merr(m, WF_ERR_CAPACITY, "streams [%d, %d) exceed max_streams %d", b->first_stream,
                    b->first_stream + b->n_streams, m->cfg.max_streams);
    if(b->n_streams == 0 || b->n_ticks == 0)
        return WF_OK;
    if(!b->pcm)
        return merr(m, WF_ERR_INVALID_ARG, "pcm is null");
    if(b->stream_stride < 0 || b->channel_stride < 0)
        return merr(m, WF_ERR_INVALID_ARG, "negative strides are not supported");
    if((long long)b->n_ticks * b->hop > 0x7fffffffLL - m->W)
        return merr(m, WF_ERR_INVALID_ARG, "n_ticks * hop too large for one call");

    WFM_CUDA(m, cudaSetDevice(m->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    const int cc = m->cfg.capture_channels, pc = m->pc, W = m->W;
    const size_t S = (size_t)b->n_streams, T = (size_t)b->n_ticks;
    const long long L = (long long)W + (long long)T * b->hop;
    int bl = kChunk;
    {
        int g = 32;
        while(g * 2 <= kChunk && (b->hop % (g * 2)) == 0 && (W % (g * 2)) == 0)
            g *= 2;
        if((b->hop % g) == 0 && (W % g) == 0)
            bl = g; // every window is a whole number of partial blocks
    }
    const int nchunk = (int)((L + kChunk - 1) / kChunk);
    const int nblk = (int)((L + bl - 1) / bl);
    const bool dev_ptrs = m_is_device_ptr(b->pcm);
    const bool is_feed = m->cfg.mode == WF_METER_INPUT_RMS;
    const size_t out_n = S * T * (is_feed ? 1 : cc);

    int rc;
    if((rc = mensure(m, &m->d_partial, &m->partial_cap, S * pc * (size_t)nblk)))
        return rc;
    if((rc = mensure(m, &m->d_raw, &m->raw_cap, S * T * pc)))
        return rc;
    const float *d_pcm = b->pcm;
    float *d_db = b->out_db, *d_lin = b->out_lin;
    unsigned char *d_silent = b->out_silent;
    if(!dev_ptrs)
    {
        const size_t span = (S - 1) * (size_t)b->stream_stride + (size_t)(cc - 1) * (size_t)b->channel_stride +
                            T * (size_t)b->hop;
        if((rc = mensure(m, &m->s_pcm, &m->pcm_cap, span)))
            return rc;
        WFM_CUDA(m, cudaMemcpyAsync(m->s_pcm, b->pcm, span * sizeof(float), cudaMemcpyHostToDevice, st));
        d_pcm = m->s_pcm;
        if(b->out_db)
        {
            if((rc = mensure(m, &m->s_db, &m->db_cap, out_n)))
                return rc;
            d_db = m->s_db;
        }
        if(b->out_lin)
        {
            if((rc = mensure(m, &m->s_lin, &m->lin_cap, out_n)))
                return rc;
            d_lin = m->s_lin;
        }
        if(b->out_silent)
        {
            if((rc = mensure(m, &m->s_silent, &m->silent_cap, S * T)))
                return rc;
            d_silent = m->s_silent;
        }
    }

    MParams p{};
    p.pcm = d_pcm;
    p.stream_stride = b->stream_stride;
    p.channel_stride = b->channel_stride;
    const size_t slot = (size_t)b->first_stream;
    p.hist = m->d_hist[m->cur] + slot * cc * W;
    p.hist_next = m->d_hist[m->cur ^ 1] + slot * cc * W;
    p.partial = m->d_partial;
    p.raw = m->d_raw;
    p.buf = m->d_buf + slot * 2;
    p.flags = m->d_flags + slot;
    p.out_db = is_feed ? nullptr : d_db;
    p.out_lin = d_lin;
    p.out_silent = is_feed ? nullptr : d_silent;
    p.n_streams = b->n_streams;
    p.n_ticks = b->n_ticks;
    p.hop = b->hop;
    p.W = W;
    p.cc = cc;
    p.pc = pc;
    p.nblk = nblk;
    p.bl = bl;
    p.nchunk = nchunk;
    p.mode = m->cfg.mode;
    {
        wf_config gc{};
        gc.tsmoothing = m->cfg.tsmoothing;
        gc.gravity = m->cfg.gravity;
        p.g = (m->cfg.tsmoothing == WF_TSMOOTH_NONE) ? 0.0f : wf::gravity_for(gc, b->seconds);
    }
    p.g2 = 1.0f - p.g;
    p.tsmooth = m->cfg.tsmoothing != WF_TSMOOTH_NONE;
    p.fast_peaks = m->cfg.fast_peaks;
    p.floor_m10 = (float)(m->cfg.floor_db - 10);
    p.db_min = m->db_min;

    WFM_CUDA(m, cudaEventRecord(m->ev0, st));
    constexpr int kWarps = 8;
    // 128-bit loads need 16-byte aligned rows (W is a multiple of 16 samples already)
    const int vec4 = (((uintptr_t)d_pcm & 15u) == 0) && ((b->stream_stride & 3) == 0) && ((b->channel_stride & 3) == 0);
    // one-pass path: the window is a whole number of hops (meter_fused_kernel)
    const size_t fused_smem = ((size_t)pc * ((size_t)(W / b->hop) + T) + T * pc) * sizeof(float);
    const bool fused = m->use_fused && vec4 && (W % b->hop) == 0 && (b->hop % 4) == 0 && fused_smem <= 96 * 1024;
    if(fused)
    {
        p.bl = b->hop;
        p.nblk = (int)(W / b->hop + T);
        // partial state: [max_streams][pc][W/hop] x 2; usable when the previous call was a one-pass call with this hop that
        // covered every stream (a reset or a general-path call invalidates it: the ring is then reduced again)
        const size_t nbk = (size_t)(W / b->hop), need = (size_t)m->cfg.max_streams * pc * nbk;
        if(need > m->part_cap)
        {
            for(auto &q : m->d_part)
            {
                if(q)
                    cudaFree(q);
                q = nullptr;
                WFM_CUDA(m, cudaMalloc((void **)&q, need * sizeof(float)));
            }
            m->part_cap = need;
            m->part_hop = 0;
        }
        const bool whole = (b->first_stream == 0) && (b->n_streams == m->cfg.max_streams);
        p.part_in = (m->part_hop == b->hop && whole) ? m->d_part[m->part_cur] : nullptr;
        p.part_out = m->d_part[m->part_cur ^ 1] + slot * pc * nbk;
        m->part_cur ^= 1;
        m->part_hop = whole ? b->hop : 0;
        auto launch = [&](auto kernel) -> cudaError_t {
            if(fused_smem > 48 * 1024)
            {
                cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
                if(err != cudaSuccess)
                    return err;
            }
            kernel<<<(int)S, 256, fused_smem, st>>>(p);
            return cudaGetLastError();
        };
        switch(m->cfg.mode)
        {
        case WF_METER_PEAK: WFM_CUDA(m, launch(meter_fused_kernel<WF_METER_PEAK>)); break;
        case WF_METER_RMS: WFM_CUDA(m, launch(meter_fused_kernel<WF_METER_RMS>)); break;
        default: WFM_CUDA(m, launch(meter_fused_kernel<WF_METER_INPUT_RMS>)); break;
        }
        m->launches += 1;
    }
    else
    {
    m->part_hop = 0; // the general path does not maintain the block partials
    const int g1 = grid_for((long long)S * pc * nchunk, kWarps, m->sm_count), g2 = grid_for((long long)S * T * pc, kWarps, m->sm_count);
    switch(m->cfg.mode)
    {
    case WF_METER_PEAK:
        meter_block_kernel<WF_METER_PEAK><<<g1, kWarps * 32, 0, st>>>(p, vec4);
        meter_window_kernel<WF_METER_PEAK><<<g2, kWarps * 32, 0, st>>>(p);
        break;
    case WF_METER_RMS:
        meter_block_kernel<WF_METER_RMS><<<g1, kWarps * 32, 0, st>>>(p, vec4);
        meter_window_kernel<WF_METER_RMS><<<g2, kWarps * 32, 0, st>>>(p);
        break;
    default:
        meter_block_kernel<WF_METER_INPUT_RMS><<<g1, kWarps * 32, 0, st>>>(p, vec4);
        meter_window_kernel<WF_METER_INPUT_RMS><<<g2, kWarps * 32, 0, st>>>(p);
        break;
    }
    WFM_CUDA(m, cudaGetLastError());
    meter_scan_kernel<<<(int)((S + 127) / 128), 128, 0, st>>>(p);
    WFM_CUDA(m, cudaGetLastError());
    m->launches += 3;
    }
    WFM_CUDA(m, cudaEventRecord(m->ev1, st));
    m->ev_valid = true;
    // The ring is double-buffered per ENGINE, so a call must cover every stream whose history should survive: copy the
    // untouched streams' rings across before flipping (cheap: only when a call addresses a subset of the streams).
    if(b->n_streams != m->cfg.max_streams)
    {
        const size_t per = (size_t)cc * W * sizeof(float);
        if(slot > 0)
            WFM_CUDA(m, cudaMemcpyAsync(m->d_hist[m->cur ^ 1], m->d_hist[m->cur], slot * per, cudaMemcpyDeviceToDevice, st));
        const size_t after = slot + S;
        if(after < (size_t)m->cfg.max_streams)
            WFM_CUDA(m, cudaMemcpyAsync(m->d_hist[m->cur ^ 1] + after * cc * W, m->d_hist[m->cur] + after * cc * W,
                                        ((size_t)m->cfg.max_streams - after) * per, cudaMemcpyDeviceToDevice, st));
    }
    m->cur ^= 1;
    if(!dev_ptrs)
    {
        if(b->out_db && !is_feed)
            WFM_CUDA(m, cudaMemcpyAsync(b->out_db, d_db, out_n * sizeof(float), cudaMemcpyDeviceToHost, st));
        if(b->out_lin)
            WFM_CUDA(m, cudaMemcpyAsync(b->out_lin, d_lin, out_n * sizeof(float), cudaMemcpyDeviceToHost, st));
        if(b->out_silent && !is_feed)
            WFM_CUDA(m, cudaMemcpyAsync(b->out_silent, d_silent, S * T, cudaMemcpyDeviceToHost, st));
    }
    return WF_OK;
}

int wf_meter_process(wf_meter *m, const wf_meter_batch *b)
{
    int rc = wf_meter_process_async(m, b, nullptr);
    if(rc)
        return rc;
    WFM_CUDA(m, cudaStreamSynchronize(m->stream));
    return WF_OK;
}

int wf_meter_reset(wf_meter *m, int32_t first, int32_t count)
{
    if(!m)
        return WF_ERR_INVALID_ARG;
    if(first < 0 || count < 0 || (int64_t)first + count > m->cfg.max_streams)
        return merr(m, WF_ERR_CAPACITY, "reset range out of bounds");
    if(count == 0)
        return WF_OK;
    WFM_CUDA(m, cudaSetDevice(m->device));
    m->part_hop = 0; // the ring of some streams is zeroed: their block partials are reduced from it again on the next call
    meter_reset_kernel<<<std::min(count, m->sm_count * 4), 256, 0, m->stream>>>(m->d_hist[m->cur], m->d_buf, m->d_flags, first,
                                                                             count, m->cfg.capture_channels, m->W);
    WFM_CUDA(m, cudaGetLastError());
    m->launches++;
    WFM_CUDA(m, cudaStreamSynchronize(m->stream));
    return WF_OK;
}

int64_t wf_meter_launch_count(const wf_meter *m) { return m ? m->launches : 0; }

float wf_meter_last_kernel_ms(wf_meter *m)
{
    if(!m || !m->ev_valid || cudaEventSynchronize(m->ev1) != cudaSuccess)
        return -1.0f;
    float ms = -1.0f;
    if(cudaEventElapsedTime(&ms, m->ev0, m->ev1) != cudaSuccess)
        return -1.0f;
    return ms;
}

} // extern "C"
