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
// Which half of a stream's ring holds its history is the stream's parity byte on the device (par): the kernels read it and the
// call's last kernel flips it, so that a call replayed from a CUDA graph reads and writes the right halves, and a call on a
// subset of the streams leaves the others' rings where they are.
// The kernels that read PCM take its sample type (float or int16_t, wf_meter_batch.pcm_format) as their last template
// argument and load it only through Pcm<TS> (wf_pcm.cuh).  The ring and the partials hold float whatever the input: an int16
// call widens its samples as it loads them, sums them in the float call's order, and leaves the state a float call leaves.
// There is no CPU fallback.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <string>
#include <vector>

#include "wf_display.cuh"
#include "wf_host.hpp"
#include "wf_splice.hpp"
#include "wf_nvtx.hpp"
#include "wf_pcm.cuh"
#include "wf_tables.hpp"
#include "wfstft.h"

namespace {

constexpr int kChunk = 256; // samples one warp reduces in K1 (8 per lane); partial blocks are 32..256 samples

struct MParams {
    const float *pcm;
    long long stream_stride, channel_stride;
    float *ring[2];      // [streams][cc][W] time-ordered ring halves: ring[par[s]] before this call, ring[par[s] ^ 1] after it
    unsigned char *par;  // [streams] parity of each stream's ring, flipped by the call's last kernel
    float *partial;      // [streams][pc][nblk]
    float *part;         // one-pass path: [streams][part_stride] the ring's block partials ([pc][W/hop] at the start of each
                         // stream's row), valid for a stream while its ptag == tag
    long long part_stride; // floats per stream of part: fixed for the buffer's allocation, whatever the call's hop
    long long *ptag;     // [streams] what the stream's partials were made for (0: none; the general path and resets clear it)
    long long tag;       // one-pass path: (generation of the partials buffer << 32) | hop
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
    // display stage (render_bars in meter mode), or null outputs
    float *out_pixels, *out_min;
    float ceiling_f, dbrange_f, px_lo, px_hi, px_cpos;
};

// render_bars in meter mode (src/source.cpp:1505-1509, :1548-1557): the bar height of each capture channel from its
// m_meter_val (val0, val1 for c < cc) and the first strict minimum starting from (cpos, 0); `st` = s * n_ticks + t
__device__ __forceinline__ void meter_pixels(const MParams &p, size_t st, float val0, float val1, int cc)
{
    float miny = p.px_cpos, minpos = 0.0f;
    for(int c = 0; c < cc; ++c)
    {
        const float v = wf::display_pixel(c ? val1 : val0, p.ceiling_f, p.dbrange_f, p.px_lo, p.px_hi);
        if(p.out_pixels)
            p.out_pixels[st * cc + c] = v;
        if(v < miny)
        {
            miny = v;
            minpos = (float)c;
        }
    }
    if(p.out_min)
    {
        p.out_min[2 * st] = miny;
        p.out_min[2 * st + 1] = minpos;
    }
}

// The ring half of stream s before this call (next = false) or after it (next = true), for the stream's parity `par`
__device__ __forceinline__ float *ring_of(const MParams &p, int s, unsigned par, bool next)
{
    return p.ring[par ^ (next ? 1u : 0u)] + (size_t)s * p.cc * p.W;
}
__device__ __forceinline__ float *ring_of(const MParams &p, int s, bool next) { return ring_of(p, s, p.par[s], next); }

// Row pointers of one (stream, channel): history ring first (timeline positions [0, W)), then this call's PCM.
template<typename TS>
struct Row {
    const float *hist;
    const TS *pcm;
};
template<typename TS>
__device__ __forceinline__ Row<TS> row_of(const MParams &p, int s, int c, unsigned par)
{
    return {ring_of(p, s, par, false) + (size_t)c * p.W,
            wf::Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride + (size_t)c * p.channel_stride};
}
template<typename TS>
__device__ __forceinline__ Row<TS> row_of(const MParams &p, int s, int c)
{
    return row_of<TS>(p, s, c, p.par[s]);
}
template<typename TS>
__device__ __forceinline__ float vsample(const Row<TS> &r, int W, long long u)
{
    return (u < W) ? r.hist[u] : wf::Pcm<TS>::ldg1(r.pcm + (u - W));
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
template<int MODE, typename TS>
__device__ __forceinline__ float reduce_range(const Row<TS> &r0, const Row<TS> &r1, bool two, int W, long long lo, long long hi,
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
// bl/8 lanes combine into one partial per bl-sample block.  Chunks that lie wholly inside new PCM aligned to 4 samples (all
// but the few that touch the history ring or the end) take two 4-sample loads per lane (128-bit for float, 64-bit for
// int16) and sum them as a pairwise tree; the others load and sum their 8 samples in sequence.  The same pass writes the last
// W samples of the timeline into the ring for the next call (every sample is read exactly once here).
template<int MODE, typename TS>
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
        // the stream's parity is loaded only by the chunks that read the ring or write the next one
        const unsigned par = (u0 < p.W || u0 + kChunk > tail0) ? p.par[s] : 0u;
        const Row<TS> r0 = row_of<TS>(p, s, c, par);
        const Row<TS> r1 = two ? row_of<TS>(p, s, 1, par) : r0;
        float *h0 = ring_of(p, s, par, true) + (size_t)c * p.W;
        float *h1 = ring_of(p, s, par, true) + (size_t)p.W;
        float acc = 0.0f;
        const long long ul = u0 + 8 * lane; // my 8 samples
        if(vec4 && u0 >= p.W && u0 + kChunk <= L)
        {
            using Quad = typename wf::Pcm<TS>::Quad;
            const Quad *q0 = reinterpret_cast<const Quad *>(r0.pcm + (ul - p.W));
            const float4 a = wf::Pcm<TS>::ldg4(q0), b = wf::Pcm<TS>::ldg4(q0 + 1);
            float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = a1;
            if(two)
            {
                const Quad *q1 = reinterpret_cast<const Quad *>(r1.pcm + (ul - p.W));
                a1 = wf::Pcm<TS>::ldg4(q1);
                b1 = wf::Pcm<TS>::ldg4(q1 + 1);
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
template<int MODE, typename TS>
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
        const unsigned par = (lo < p.W) ? p.par[s] : 0u; // only windows that reach into the ring read it
        const Row<TS> r0 = row_of<TS>(p, s, c, par);
        const Row<TS> r1 = two ? row_of<TS>(p, s, 1, par) : r0;
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

// K3: one thread per stream, the per-tick recurrence (src/source_generic.cpp:232-269).  K1 and K2 are done with the ring:
// the stream's parity flips, and its block partials (which K1 does not keep) are no longer valid.
__global__ void meter_scan_kernel(const MParams p)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if(s >= p.n_streams)
        return;
    p.par[s] ^= 1;
    p.ptag[s] = 0;
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
        float val0 = 0.0f, val1 = 0.0f;
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
            (c ? val1 : val0) = val;
            const size_t o = ((size_t)s * p.n_ticks + t) * p.cc + c;
            if(p.out_db)
                p.out_db[o] = val;
            if(p.out_lin)
                p.out_lin[o] = out;
        }
        last_silent = silent_channels >= p.cc; // :264-269
        if(p.out_pixels || p.out_min)
            meter_pixels(p, (size_t)s * p.n_ticks + t, val0, val1, p.cc);
        if(p.out_silent)
            p.out_silent[(size_t)s * p.n_ticks + t] = last_silent ? 1 : 0;
    }
    p.buf[2 * s] = buf[0];
    p.buf[2 * s + 1] = buf[1];
    p.flags[s] = last_silent ? 1 : 0;
}

// ---- one-pass path: hop divides the window (the plugin's usual case: 150 ms at 48 kHz = 7200 = 9 x 800 samples at 60 fps) ----
// One CTA per stream.  Every hop-sized block of the stream's timeline (W/hop blocks of history ring, then one block per
// tick) is reduced ONCE by one warp with 4-sample loads — the same pass copies the last W samples into the next call's ring —
// and its partial lands in shared memory; a tick's window is then exactly W/hop consecutive partials, combined by one
// thread per (tick, channel); finally the per-stream recurrence (EMA, dBFS, m_last_silent) runs on one lane per channel.
// Samples cross HBM once, nothing else does: the three-kernel path above wrote and re-read per-32-sample partials W/hop times.
// A lane's groups of 4 samples are i0 + 32u whatever the sample type: int16 blocks take 64-bit loads in the same grouping.
template<int MODE, typename TS>
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
    const bool have_part = p.ptag[s] == p.tag;
    if(have_part)
        for(int i = threadIdx.x; i < pc * nb; i += blockDim.x)
            part[(i / nb) * NB + (i % nb)] = p.part[(size_t)s * p.part_stride + i];
    for(int w = warp; w < pc * NB; w += nwarps)
    {
        const int c = w / NB, b = w - c * NB;
        if(have_part && b < nb && b < T)
            continue;
        const Row<TS> r0 = row_of<TS>(p, s, c);
        const Row<TS> r1 = two ? row_of<TS>(p, s, 1) : r0;
        // block b: the ring (float, read as float4) for b < nb, else this call's PCM (read as Pcm<TS>::Quad); group i is
        // samples [4i, 4i+4) of the block either way
        using Quad = typename wf::Pcm<TS>::Quad;
        const Quad *src0 = reinterpret_cast<const Quad *>((b < nb) ? reinterpret_cast<const TS *>(r0.hist + (size_t)b * hop)
                                                                   : r0.pcm + (size_t)(b - nb) * hop);
        const Quad *src1 = reinterpret_cast<const Quad *>((b < nb) ? reinterpret_cast<const TS *>(r1.hist + (size_t)b * hop)
                                                                   : r1.pcm + (size_t)(b - nb) * hop);
        const bool keep = b >= T; // one of the last W/hop blocks: belongs to the next call's ring
        float4 *h0 = reinterpret_cast<float4 *>(ring_of(p, s, true) + (size_t)c * W + (size_t)(b - T) * hop);
        float4 *h1 = reinterpret_cast<float4 *>(ring_of(p, s, true) + (size_t)W + (size_t)(b - T) * hop);
        float acc = 0.0f;
        // four loads in flight per lane and channel, 128-bit for float and 64-bit for int16 (a hop of 800 samples is 6.25 loads
        // per lane; eight int16 loads in flight cost registers and occupancy and were slower)
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
                    a[u] = (b < nb) ? reinterpret_cast<const float4 *>(src0)[i] : wf::Pcm<TS>::ldg4(src0 + i);
                    if(two)
                        a1[u] = (b < nb) ? reinterpret_cast<const float4 *>(src1)[i] : wf::Pcm<TS>::ldg4(src1 + i);
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
    __syncthreads(); // every read of the ring, its parity and the stream's partials is behind this barrier
    for(int i = threadIdx.x; i < pc * nb; i += blockDim.x) // the ring's partials for the next call
        p.part[(size_t)s * p.part_stride + i] = part[(i / nb) * NB + T + (i % nb)];
    if(threadIdx.x == 0)
    {
        p.par[s] ^= 1;
        p.ptag[s] = p.tag;
    }
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
        float val0 = 0.0f, val1 = 0.0f;
        for(int c = 0; c < cc; ++c)
        {
            const float out = raw[t * pc + c];
            const float val = (out > 0.0f) ? 20.0f * log10f(out) : p.db_min; // dbfs, src/source.hpp:293-299
            below += (val < p.floor_m10) ? 1 : 0;
            (c ? val1 : val0) = val;
            const size_t o = ((size_t)s * T + t) * cc + c;
            if(p.out_db)
                p.out_db[o] = val;
            if(p.out_lin)
                p.out_lin[o] = out;
        }
        const bool silent = below >= cc; // :264-269
        if(p.out_pixels || p.out_min)
            meter_pixels(p, (size_t)s * T + t, val0, val1, cc);
        if(p.out_silent)
            p.out_silent[(size_t)s * T + t] = silent ? 1 : 0;
        if(t == T - 1)
            p.flags[s] = silent ? 1 : 0;
    }
}

// timeout branch (src/source_generic.cpp:184-199) for streams [first, first+count); their block partials are reduced from
// the ring again on the next call
__global__ void meter_reset_kernel(float *ring0, float *ring1, const unsigned char *par, long long *ptag, float *buf,
                                   unsigned char *flags, int first, int count, int cc, int W)
{
    for(int s = first + blockIdx.x; s < first + count; s += gridDim.x)
    {
        if(threadIdx.x == 0)
            ptag[s] = 0;
        if(flags[s] != 0)
            continue; // already silent: tick returns early
        float *hist = par[s] ? ring1 : ring0;
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

// wf_meter_get_state / wf_meter_set_state: the state of streams [first, first+count) between the device layouts and the
// sections of one staging buffer (x_*, null = skipped), one CTA per stream.  The ring is the half the stream's parity
// selects, read here because after graph replays only the device knows it.  SET also drops the stream's block partials
// (as a reset does): the next one-pass call reduces the restored ring again, block by block in the order it reduced those
// samples as new PCM, so it gets the partials the stream's history would have left bit for bit.
struct MStateIO {
    float *ring[2];
    const unsigned char *par;
    long long *ptag;
    float *buf, *line;
    unsigned char *flags;
    float *x_ring, *x_line, *x_ema; // [count][cc][W], [count][cc][D], [count][cc]
    unsigned char *x_flags;         // [count]
    int first, count, cc, W, D;
};
template<bool SET>
__device__ __forceinline__ void move_state(float *dev, float *x, long long n)
{
    for(long long k = threadIdx.x; k < n; k += blockDim.x)
    {
        if(SET)
            dev[k] = x[k];
        else
            x[k] = dev[k];
    }
}
template<bool SET>
__global__ void meter_state_kernel(const MStateIO q)
{
    for(int i = blockIdx.x; i < q.count; i += gridDim.x)
    {
        const int s = q.first + i;
        const long long rn = (long long)q.cc * q.W, ln = (long long)q.cc * q.D;
        if(q.x_ring)
            move_state<SET>(((q.par[s] & 1) ? q.ring[1] : q.ring[0]) + (size_t)s * rn, q.x_ring + (size_t)i * rn, rn);
        if(q.x_line)
            move_state<SET>(q.line + (size_t)s * ln, q.x_line + (size_t)i * ln, ln);
        if(q.x_ema)
            move_state<SET>(q.buf + 2 * (size_t)s, q.x_ema + (size_t)i * q.cc, q.cc);
        if(threadIdx.x == 0)
        {
            if(q.x_flags)
            {
                if(SET)
                    q.flags[s] = q.x_flags[i] & 1;
                else
                    q.x_flags[i] = q.flags[s] & 1;
            }
            if(SET)
                q.ptag[s] = 0;
        }
    }
}

// The kernels of one mode and sample type: the one-pass kernel, and K1 and K2 of the three-kernel path (K3,
// meter_scan_kernel, reads no PCM and has one instantiation)
struct MeterKernels {
    void (*fused)(MParams);
    void (*block)(MParams, int);
    void (*window)(MParams);
};
template<int MODE>
constexpr MeterKernels kMeterKernels[2] = { // [s16]
    {meter_fused_kernel<MODE, float>, meter_block_kernel<MODE, float>, meter_window_kernel<MODE, float>},
    {meter_fused_kernel<MODE, int16_t>, meter_block_kernel<MODE, int16_t>, meter_window_kernel<MODE, int16_t>}};

} // namespace

struct wf_meter : wf::HostCore {
    wf_meter_config cfg{};
    int W = 0, pc = 1;
    float db_min = 0.0f;
    wf::DevBuf<float> d_hist[2];
    wf::DevBuf<unsigned char> d_par; // [max_streams] which half of d_hist holds each stream's ring (MParams::par)
    // one-pass path: block partials of the ring [max_streams][pc * part_nbk] and what each stream's were made for
    // (MParams::ptag).  Each stream's row has room for the most blocks (W/hop) any call has needed, so a call with one hop
    // never writes into another stream's row; part_gen counts the buffer's layouts (allocations), so that partials of an
    // earlier layout never pass for the current one's
    wf::DevBuf<float> d_part;
    wf::DevBuf<long long> d_ptag;
    long long part_gen = 0;
    int part_nbk = 0;
    bool use_fused = true; // WF_METER_FUSED=0: always the three-kernel path (A/B tests)
    const MeterKernels *kern = nullptr; // [s16]: the instantiations of the engine's mode
    wf::DevBuf<float> d_buf;
    wf::DevBuf<unsigned char> d_flags;
    // audio sync offset: the newest D samples of each stream slot and capture channel, held back for the next call
    int D = 0;
    wf::DevBuf<float> d_line;   // [max_streams][cc][D], zeros at creation
    wf::DevBuf<float> s_window; // (line ++ new) of a call, in its sample type (counts floats)
    // scratch / staging
    wf::DevBuf<float> d_partial, d_raw, s_pcm, s_db, s_lin, s_pixels, s_min;
    wf::DevBuf<unsigned char> s_silent;
    // wf_meter_get_state / wf_meter_set_state: the sections of a call, on the device and on the host
    wf::DevBuf<unsigned char> s_state;
    std::vector<unsigned char> h_state;
    // display stage: only when the config carried display settings (current struct size)
    bool display = false;
    float ceiling_f = 0.0f, dbrange_f = 1.0f, px_lo = 0.0f, px_hi = 0.0f, px_cpos = 0.0f;
};

namespace {

thread_local std::string g_meter_create_error;

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
    c->height = 225;
    c->ceiling_db = 0;
    c->bar_width = 24;
    c->rounded_caps = 0;
    c->min_bar_height = 0;
    c->sync_offset_ms = 0;
}

const char *wf_meter_last_error(const wf_meter *m) { return m ? m->last_error.c_str() : g_meter_create_error.c_str(); }

int wf_meter_create(const wf_meter_config *cfg_in, wf_meter **out)
{
    if(!cfg_in || !out)
        return WF_ERR_INVALID_ARG;
    *out = nullptr;
    return wf::create_engine(out, g_meter_create_error, wf_meter_destroy, [&](wf_meter *m) -> int {
        // the current struct, the previous one (which ends before sync_offset_ms: no offset) or the one before (which ends
        // before height: its display settings are absent)
        bool current = false;
        if(!wf::accept_struct(cfg_in, {offsetof(wf_meter_config, sync_offset_ms), offsetof(wf_meter_config, height)}, m->cfg,
                              &current))
            return wf::fail(m, WF_ERR_ABI, "wf_meter_config.struct_size mismatch");
        const bool display_settings = current || cfg_in->struct_size == offsetof(wf_meter_config, sync_offset_ms);
        const wf_meter_config *cfg = &m->cfg;
        if(!wf::sync_offset_ok(cfg->sync_offset_ms))
            return wf::fail(m, WF_ERR_INVALID_ARG, "sync_offset_ms %d outside [-1000, 1000]", cfg->sync_offset_ms);
        if(cfg->capture_channels < 1 || cfg->capture_channels > 2 || cfg->max_streams < 1 || cfg->sample_rate < 16 ||
           cfg->mode < WF_METER_PEAK || cfg->mode > WF_METER_INPUT_RMS)
            return wf::fail(m, WF_ERR_INVALID_ARG, "bad meter config");
        int W;
        if(cfg->mode == WF_METER_INPUT_RMS)
            W = (int)(cfg->sample_rate & ~15u); // m_input_rms_size, src/source.cpp:1148
        else
            W = (int)(((size_t)((double)cfg->sample_rate * ((double)cfg->meter_ms / 1000.0))) & ~(size_t)15); // :1121
        if(W < 16)
            return wf::fail(m, WF_ERR_INVALID_ARG, "meter window of %d ms is shorter than 16 samples", cfg->meter_ms);
        if(int rc = wf::open_device(m, cfg->device))
            return rc;
        m->W = W;
        m->pc = (cfg->mode == WF_METER_INPUT_RMS) ? 1 : cfg->capture_channels;
        m->db_min = 20.0f * log10f(1.17549435e-38f); // DB_MIN, src/source.cpp:43
        m->display = display_settings && cfg->mode != WF_METER_INPUT_RMS;
        if(m->display)
        {
            // render_bars geometry in meter mode (src/source.cpp:1481-1494; m_stereo is forced off, :1115, so cpos = height and
            // the channel spacing is 0) after the get_settings clamps (:573-577) and m_cap_radius = bar_width / 2 (:1297)
            int ceiling = cfg->ceiling_db, floor = cfg->floor_db;
            if((ceiling - floor) < 1)
            {
                ceiling = 0;
                floor = -120;
            }
            const float cpos = (float)(cfg->height < 1 ? 225 : cfg->height);
            const float cap_radius = (float)cfg->bar_width / 2.0f;
            const float border_top = cfg->rounded_caps ? cap_radius : 0.0f;
            float border_bottom = cfg->rounded_caps ? cpos - cap_radius : cpos;
            if(cfg->min_bar_height > 0)
                border_bottom -= cfg->min_bar_height;
            border_bottom = std::clamp(border_bottom, border_top, cpos);
            m->ceiling_f = (float)ceiling;
            m->dbrange_f = (float)(ceiling - floor);
            m->px_lo = border_top;
            m->px_hi = border_bottom;
            m->px_cpos = cpos;
        }
        m->use_fused = wf::env_flag("WF_METER_FUSED", true);
        m->kern = (cfg->mode == WF_METER_PEAK) ? kMeterKernels<WF_METER_PEAK>
                  : (cfg->mode == WF_METER_RMS) ? kMeterKernels<WF_METER_RMS>
                                                 : kMeterKernels<WF_METER_INPUT_RMS>;
        const size_t S = (size_t)cfg->max_streams, hist_n = S * cfg->capture_channels * (size_t)W;
        int rc;
        for(auto &h : m->d_hist)
            if((rc = h.reserve(m, hist_n)))
                return rc;
        if((rc = m->d_buf.reserve(m, S * 2)))
            return rc;
        if((rc = m->d_flags.reserve(m, S)))
            return rc;
        if((rc = m->d_par.reserve(m, S)) || (rc = m->d_ptag.reserve(m, S)))
            return rc;
        WF_CHECK(m, cudaMemsetAsync(m->d_par, 0, S, m->stream));
        WF_CHECK(m, cudaMemsetAsync(m->d_ptag, 0, S * sizeof(long long), m->stream));
        m->D = wf::sync_delay(cfg->sample_rate, cfg->sync_offset_ms);
        if(m->D > 0)
        {
            const size_t line_n = S * cfg->capture_channels * (size_t)m->D;
            if((rc = m->d_line.reserve(m, line_n)))
                return rc;
            WF_CHECK(m, cudaMemsetAsync(m->d_line, 0, line_n * sizeof(float), m->stream));
        }
        // ≙ update(): ring := 0 (src/source.cpp:1181), m_meter_buf := DB_MIN (:1124-1125, sic), m_last_silent := false (:1236)
        WF_CHECK(m, cudaMemsetAsync(m->d_hist[0], 0, hist_n * sizeof(float), m->stream));
        WF_CHECK(m, cudaMemsetAsync(m->d_flags, 0, S, m->stream));
        if((rc = wf::fill_device(m, m->d_buf, (long long)S * 2, m->db_min, m->stream)))
            return rc;
        WF_CHECK(m, cudaStreamSynchronize(m->stream));
        return WF_OK;
    });
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
    delete m;
}

int32_t wf_meter_window(const wf_meter *m) { return m ? m->W : 0; }

int wf_meter_process_async(wf_meter *m, const wf_meter_batch *b_in, void *cuda_stream)
{
    if(!m || !b_in)
        return WF_ERR_INVALID_ARG;
    wf::NvtxRange nvtx("wf_meter_process");
    // the current struct, the previous one (which ends before pcm_format: float PCM) or the one before (which ends before
    // out_pixels: no display outputs either)
    wf_meter_batch bv;
    if(!wf::accept_struct(b_in, {offsetof(wf_meter_batch, pcm_format), offsetof(wf_meter_batch, out_pixels)}, bv))
        return wf::fail(m, WF_ERR_ABI, "wf_meter_batch.struct_size %u != %zu", b_in->struct_size, sizeof(wf_meter_batch));
    const wf_meter_batch *b = &bv;
    if((b->out_pixels || b->out_min) && !m->display)
        return wf::fail(m, WF_ERR_INVALID_ARG, (m->cfg.mode == WF_METER_INPUT_RMS)
                                               ? "display outputs do not exist for the RMS feed (INPUT_RMS)"
                                               : "display outputs need an engine created with display settings");
    if(b->n_streams < 0 || b->n_ticks < 0 || b->hop < 1)
        return wf::fail(m, WF_ERR_INVALID_ARG, "n_streams/n_ticks must be >= 0 and hop >= 1");
    if(int rc = wf::check_slot_range(m, b->first_stream, b->n_streams, m->cfg.max_streams, "stream"))
        return rc;
    if(b->n_streams == 0 || b->n_ticks == 0)
        return WF_OK;
    if(!b->pcm)
        return wf::fail(m, WF_ERR_INVALID_ARG, "pcm is null");
    wf::PcmBatch pb;
    if(int rc = wf::check_pcm_batch(m, *b, m->cfg.capture_channels, m->W, &pb))
        return rc;

    WF_CHECK(m, cudaSetDevice(m->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    WF_CHECK(m, wf::begin_call(m, st));
    if(int rc = wf::refuse_pageable(m, {b->pcm, b->out_db, b->out_lin, b->out_silent, b->out_pixels, b->out_min}))
        return rc;
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
    const bool is_feed = m->cfg.mode == WF_METER_INPUT_RMS;
    const size_t out_n = S * T * (is_feed ? 1 : cc);

    int rc;
    if((rc = m->d_partial.reserve(m, S * pc * (size_t)nblk)))
        return rc;
    if((rc = m->d_raw.reserve(m, S * T * pc)))
        return rc;
    // a call with host buffers (told by pcm alone) is staged through device memory; the RMS feed has no dB / silent outputs
    wf::Staging io(m, st, !wf::is_device_ptr(b->pcm));
    wf::PcmView pcm{io.in_bytes(m->s_pcm, b->pcm, pb.span * pb.sample_bytes), b->stream_stride, b->channel_stride};
    float *d_db = io.out(m->s_db, is_feed ? nullptr : b->out_db, out_n);
    float *d_lin = io.out(m->s_lin, b->out_lin, out_n);
    unsigned char *d_silent = io.out(m->s_silent, is_feed ? nullptr : b->out_silent, S * T);
    float *d_pixels = io.out(m->s_pixels, b->out_pixels, out_n);
    float *d_min = io.out(m->s_min, b->out_min, S * T * 2);
    if(io.rc)
        return io.rc;

    const size_t slot = (size_t)b->first_stream;
    WF_CHECK(m, wf::time_begin(m, st));
    // with a sync offset the kernels read (line ++ new)[0 .. T*hop) and the line keeps the last D samples (wf_splice.hpp)
    if(m->D > 0)
    {
        const long long tl = (long long)T * b->hop;
        if((rc = wf::splice_holdback(m, m->d_line + slot * cc * m->D, m->D, (int)S, cc, tl, std::max<long long>(tl, m->D),
                                     pb.s16, m->s_window, pcm, st)))
            return rc;
    }

    MParams p{};
    p.pcm = pcm.pcm;
    p.stream_stride = pcm.stream_stride;
    p.channel_stride = pcm.channel_stride;
    p.ring[0] = m->d_hist[0] + slot * cc * W;
    p.ring[1] = m->d_hist[1] + slot * cc * W;
    p.par = m->d_par + slot;
    p.ptag = m->d_ptag + slot;
    p.partial = m->d_partial;
    p.raw = m->d_raw;
    p.buf = m->d_buf + slot * 2;
    p.flags = m->d_flags + slot;
    p.out_db = d_db;
    p.out_lin = d_lin;
    p.out_silent = d_silent;
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
    p.out_pixels = d_pixels;
    p.out_min = d_min;
    p.ceiling_f = m->ceiling_f;
    p.dbrange_f = m->dbrange_f;
    p.px_lo = m->px_lo;
    p.px_hi = m->px_hi;
    p.px_cpos = m->px_cpos;

    constexpr int kWarps = 8;
    // 4-sample group loads (128-bit for float, 64-bit for int16) need rows aligned to 4 samples (W is a multiple of 16
    // samples already).  The facts are stated in samples, so an int16 call takes the float call's path and summation order.
    const int vec4 = (((uintptr_t)pcm.pcm & (4 * pb.sample_bytes - 1)) == 0) && ((pcm.stream_stride & 3) == 0) &&
                     ((pcm.channel_stride & 3) == 0);
    // one-pass path: the window is a whole number of hops (meter_fused_kernel)
    const size_t fused_smem = ((size_t)pc * ((size_t)(W / b->hop) + T) + T * pc) * sizeof(float);
    const bool fused = m->use_fused && vec4 && (W % b->hop) == 0 && (b->hop % 4) == 0 && fused_smem <= 96 * 1024;
    const MeterKernels &k = m->kern[pb.s16];
    if(fused)
    {
        p.bl = b->hop;
        p.nblk = (int)(W / b->hop + T);
        // a stream's partials are usable when its last call was a one-pass call with this hop into this buffer (a reset or a
        // general-path call invalidates them: the ring is then reduced again)
        if(W / b->hop > m->part_nbk)
        {
            m->part_nbk = W / b->hop;
            ++m->part_gen; // a new layout, allocated below: no partials yet
        }
        p.part_stride = (long long)pc * m->part_nbk;
        if((rc = m->d_part.reserve(m, (size_t)m->cfg.max_streams * p.part_stride)))
            return rc;
        p.part = m->d_part + slot * p.part_stride;
        p.tag = (m->part_gen << 32) | b->hop;
        WF_CHECK(m, wf::launch_kernel(k.fused, m->device, (unsigned)S, 256, fused_smem, st, {}, p));
        m->launches += 1;
    }
    else
    {
        const int g1 = grid_for((long long)S * pc * nchunk, kWarps, m->sm_count);
        const int g2 = grid_for((long long)S * T * pc, kWarps, m->sm_count);
        WF_CHECK(m, wf::launch_kernel(k.block, m->device, g1, kWarps * 32, 0, st, {}, p, vec4));
        WF_CHECK(m, wf::launch_kernel(k.window, m->device, g2, kWarps * 32, 0, st, {}, p));
        WF_CHECK(m, wf::launch_kernel(meter_scan_kernel, m->device, (unsigned)((S + 127) / 128), 128, 0, st, {}, p));
        m->launches += 3;
    }
    WF_CHECK(m, wf::time_end(m, st));
    return io.finish();
}

int wf_meter_process(wf_meter *m, const wf_meter_batch *b)
{
    int rc = wf_meter_process_async(m, b, nullptr);
    if(rc)
        return rc;
    WF_CHECK(m, cudaStreamSynchronize(m->stream));
    return WF_OK;
}

int wf_meter_reset(wf_meter *m, int32_t first, int32_t count)
{
    if(!m)
        return WF_ERR_INVALID_ARG;
    if(int rc = wf::check_slot_range(m, first, count, m->cfg.max_streams, "reset"))
        return rc;
    if(count == 0)
        return WF_OK;
    WF_CHECK(m, cudaSetDevice(m->device));
    WF_CHECK(m, wf::launch_kernel(meter_reset_kernel, m->device, std::min(count, m->sm_count * 4), 256, 0, m->stream, {},
                                  m->d_hist[0].p, m->d_hist[1].p, m->d_par.p, m->d_ptag.p, m->d_buf.p, m->d_flags.p, first,
                                  count, m->cfg.capture_channels, m->W));
    m->launches++;
    WF_CHECK(m, cudaStreamSynchronize(m->stream));
    return WF_OK;
}

} // extern "C"

namespace {

// wf_meter_get_state (set = false) / wf_meter_set_state (set = true): the range check, then one copy and one launch on the
// engine's stream, which is synchronised
int meter_state(wf_meter *m, int32_t first, int32_t count, const float *ring, const float *line, const float *ema,
                const uint8_t *flags, bool set)
{
    if(!m)
        return WF_ERR_INVALID_ARG;
    if(int rc = wf::check_slot_range(m, first, count, m->cfg.max_streams, "state"))
        return rc;
    const size_t n = (size_t)count, cc = (size_t)m->cfg.capture_channels;
    wf::StateSections io;
    const int i_ring = io.add(ring, n * cc * m->W * sizeof(float));
    const int i_line = io.add(line, n * cc * m->D * sizeof(float));
    const int i_ema = io.add((m->cfg.mode == WF_METER_INPUT_RMS) ? nullptr : ema, n * cc * sizeof(float));
    const int i_flags = io.add(flags, n);
    if(io.empty())
        return WF_OK;
    WF_CHECK(m, cudaSetDevice(m->device));
    if(int rc = io.reserve(m, m->s_state, m->h_state))
        return rc;
    MStateIO q{};
    q.ring[0] = m->d_hist[0];
    q.ring[1] = m->d_hist[1];
    q.par = m->d_par;
    q.ptag = m->d_ptag;
    q.buf = m->d_buf;
    q.line = m->d_line;
    q.flags = m->d_flags;
    q.x_ring = io.dev<float>(i_ring);
    q.x_line = io.dev<float>(i_line);
    q.x_ema = io.dev<float>(i_ema);
    q.x_flags = io.dev<unsigned char>(i_flags);
    q.first = first;
    q.count = count;
    q.cc = (int)cc;
    q.W = m->W;
    q.D = m->D;
    const int grid = std::min(count, m->sm_count * 4);
    return io.run(m, m->stream, set, [&] {
        const cudaError_t err = wf::launch_kernel(set ? meter_state_kernel<true> : meter_state_kernel<false>, m->device,
                                                  grid, 256, 0, m->stream, {}, q);
        m->launches += (err == cudaSuccess);
        return err;
    });
}

} // namespace

extern "C" {

int wf_meter_get_state(wf_meter *m, int32_t first, int32_t count, float *ring, float *line, float *ema, uint8_t *flags)
{
    return meter_state(m, first, count, ring, line, ema, flags, false);
}

int wf_meter_set_state(wf_meter *m, int32_t first, int32_t count, const float *ring, const float *line, const float *ema,
                       const uint8_t *flags)
{
    return meter_state(m, first, count, ring, line, ema, flags, true);
}

int64_t wf_meter_launch_count(const wf_meter *m) { return m ? m->launches : 0; }

float wf_meter_last_kernel_ms(wf_meter *m) { return wf::last_kernel_ms(m); }

} // extern "C"
