// wf_splice.cu — history ++ new splice of wf_splice.hpp, shared by the spectrum, level-meter and waveform engines, and the
// holdback call the level meter and the waveform make of it.
#include "wf_splice.hpp"

namespace wf {
namespace {

// float history sample -> the sample type of the call: an int16 call sees the history rounded to int16 (exact for a
// history that int16 calls or the start-up zeros filled)
__device__ __forceinline__ float history_sample(float x, float) { return x; }
__device__ __forceinline__ int16_t history_sample(float x, int16_t)
{
    return (int16_t)max(-32768l, min(32767l, lrintf(x * 32768.0f)));
}
__device__ __forceinline__ float widen_sample(float x) { return x; }
__device__ __forceinline__ float widen_sample(int16_t v) { return (float)v * 0x1p-15f; }

// Copies n samples, 16 bytes at a time when both ends are 16-byte aligned (the caller's layout decides), else one sample at
// a time.
template<typename TS>
__device__ __forceinline__ void copy_samples(TS *dst, const TS *src, long long n)
{
    if((((uintptr_t)dst | (uintptr_t)src) & 15u) == 0)
    {
        constexpr int V = 16 / sizeof(TS);
        const long long nv = n / V;
        for(long long i = threadIdx.x; i < nv; i += blockDim.x)
            reinterpret_cast<uint4 *>(dst)[i] = __ldg(reinterpret_cast<const uint4 *>(src) + i);
        for(long long i = nv * V + threadIdx.x; i < n; i += blockDim.x)
            dst[i] = src[i];
    }
    else
        for(long long i = threadIdx.x; i < n; i += blockDim.x)
            dst[i] = src[i];
}

// One CTA per (stream, channel):
//   0. with owed (channel 0's CTA): the stream's skip_mask of the call, then its owed count less L;
//   1. window := C[ws .. ws + wl): the history part (converted to the call's type), then the new part;
//   2. history := C[L .. L + R), read behind the barrier from the window where it covers them, else from the new samples.
// The new samples are read at most twice (window, then the history's tail beyond the window) and never beyond L.
template<typename TS>
__global__ void __launch_bounds__(256) history_splice_kernel(const Splice p)
{
    const int s = blockIdx.x, c = blockIdx.y, cc = gridDim.y, R = p.R;
    if(p.owed && c == 0)
    {
        const long long owed = p.owed[s];
        // tick t is short of audio while owed > (t+1)*hop
        const long long nskip = owed > 0 ? min((long long)p.T, (owed + p.hop - 1) / p.hop - 1) : 0;
        const size_t row = (size_t)s * p.T;
        for(int t = threadIdx.x; t < p.T; t += blockDim.x)
            p.mask[row + t] = (t < nskip) || (p.caller && p.caller[row + t]);
        __syncthreads();
        if(threadIdx.x == 0)
            p.owed[s] = max(0ll, owed - p.L);
    }
    float *hist = p.hist + ((size_t)s * cc + c) * R;
    const TS *nw = static_cast<const TS *>(p.pcm) + s * p.stream_stride + c * p.channel_stride;
    TS *win = nullptr;
    if(p.win)
    {
        win = static_cast<TS *>(p.win) + ((size_t)s * cc + c) * p.win_cs;
        const long long hw = max(0ll, min(p.wl, (long long)R - p.ws)); // window samples taken from the history
        for(long long i = threadIdx.x; i < hw; i += blockDim.x)
            win[i] = history_sample(hist[p.ws + i], TS{});
        copy_samples(win + hw, nw + (p.ws + hw - R), p.wl - hw);
        __syncthreads();
    }
    const long long wend = win ? p.ws + p.wl : 0;
    for(int i = threadIdx.x; i < R; i += blockDim.x)
    {
        const long long j = p.L + i;
        hist[i] = (j < wend) ? widen_sample(win[j - p.ws]) : widen_sample(nw[j - R]);
    }
}

} // namespace

cudaError_t launch_splice(const Splice &s, int device, int streams, int cc, bool s16, cudaStream_t st)
{
    return launch_kernel(s16 ? history_splice_kernel<int16_t> : history_splice_kernel<float>, device,
                         dim3((unsigned)streams, (unsigned)cc), 256, 0, st, {}, s);
}

int splice_holdback(HostCore *c, float *hist, int R, int streams, int cc, long long L, long long wl, bool s16,
                    DevBuf<float> &window, PcmView &view, cudaStream_t st)
{
    const long long cs = splice_stride(wl, s16);
    if(int rc = window.reserve(c, ((size_t)streams * cc * (size_t)cs * (s16 ? 2 : 4) + 3) / 4))
        return rc;
    Splice sp{};
    sp.hist = hist;
    sp.win = window.p;
    sp.pcm = view.pcm;
    sp.stream_stride = view.stream_stride;
    sp.channel_stride = view.channel_stride;
    sp.win_cs = cs;
    sp.ws = 0;
    sp.wl = wl;
    sp.L = L;
    sp.R = R;
    WF_CHECK(c, launch_splice(sp, c->device, streams, cc, s16, st));
    c->launches++;
    view = {window.p, cc * cs, cs};
    return WF_OK;
}

} // namespace wf
