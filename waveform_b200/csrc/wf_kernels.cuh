// wf_kernels.cuh — device code shared by the spectrum kernel families (no kernels): the Stockham FFT plans and passes of
// the power-of-two sizes (fused, wide), group-level votes, dBFS, and the render-time display stage.
//
// Reference semantics restated here: dbfs src/source.hpp:293-299, render-time interpolation
// src/source.cpp:1381-1406,1510-1546 + src/filter.hpp:133-211.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "wf_fft.cuh"
#include "wf_kparams.hpp"
#include "wf_pcm.cuh"
#include "wf_sm90.cuh"

namespace wf {

// ---- plans: threads per frame (TN) and per-pass radices for each supported N -----------------------
template<int TN_, int... Rs>
struct PlanT {
    using type = PlanT<TN_, Rs...>;
    static constexpr int TN = TN_;
    static constexpr int NPASS = sizeof...(Rs);
};
template<int N> struct Plan;
template<> struct Plan<128> : PlanT<8, 8, 8> {};
template<> struct Plan<256> : PlanT<8, 16, 8> {};
template<> struct Plan<512> : PlanT<16, 16, 16> {};
template<> struct Plan<1024> : PlanT<16, 32, 16> {};
template<> struct Plan<2048> : PlanT<32, 32, 32> {};
template<> struct Plan<4096> : PlanT<128, 16, 16, 8> {};
template<> struct Plan<8192> : PlanT<256, 16, 16, 16> {};
template<> struct Plan<16384> : PlanT<256, 32, 16, 16> {};
template<> struct Plan<32768> : PlanT<512, 32, 32, 16> {};

template<int N>
struct Geo {
    static constexpr int M = N / 2;
    static constexpr int TN = Plan<N>::TN;
    static constexpr int P = M / TN;                          // complex points (= bins) per thread
    static constexpr int CTA = (TN >= 128) ? TN : 128;        // threads per CTA
    static constexpr int GROUPS = CTA / TN;                   // streams per CTA
    static constexpr int BUF = M + (M >> 5);                  // padded exchange buffer, float2 elements
    // register cap: 128 registers/thread (512 threads per SM resident) — without it ptxas takes ~250 registers for
    // hoisted twiddle loads and the kernels run at 8 warps/SM
#ifndef WF_THREADS_PER_SM
#define WF_THREADS_PER_SM 512
#endif
    static constexpr int MINB = (WF_THREADS_PER_SM / CTA) > 0 ? (WF_THREADS_PER_SM / CTA) : 1;
};

__device__ __forceinline__ int phys(int i) { return i + (i >> 5); }

// ---- group-level sync / votes -----------------------------------------------------------------------
// Sub-warp groups (TN < 32: several streams share a warp) may diverge from one another (one stream is gated
// while its neighbour is not), so every warp-level primitive names only the lanes of the calling group.
template<int TN>
__device__ __forceinline__ unsigned group_mask()
{
    if constexpr(TN >= 32)
        return 0xffffffffu;
    else
    {
        const unsigned lane = threadIdx.x & 31u;
        return ((1u << TN) - 1u) << (lane & ~(unsigned)(TN - 1));
    }
}
template<int TN>
__device__ __forceinline__ void group_sync()
{
    if constexpr(TN <= 32)
        __syncwarp(group_mask<TN>());
    else
        __syncthreads();
}
template<int TN>
__device__ __forceinline__ bool group_any(bool x)
{
    if constexpr(TN <= 32)
        return __ballot_sync(group_mask<TN>(), x) != 0u;
    else
        return __syncthreads_or(x) != 0;
}
template<int TN>
__device__ __forceinline__ bool group_all(bool x)
{
    return !group_any<TN>(!x);
}
template<int TN>
__device__ __forceinline__ float group_max(float x, float *scratch)
{
    if constexpr(TN <= 32)
    {
        const unsigned m = group_mask<TN>();
#pragma unroll
        for(int o = TN / 2; o > 0; o >>= 1)
            x = fmaxf(x, __shfl_xor_sync(m, x, o));
        return x;
    }
    else
    {
#pragma unroll
        for(int o = 16; o > 0; o >>= 1)
            x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
        __syncthreads();
        if((threadIdx.x & 31) == 0)
            scratch[threadIdx.x >> 5] = x;
        __syncthreads();
        float m = scratch[0];
        for(int w = 1; w < TN / 32; ++w)
            m = fmaxf(m, scratch[w]);
        return m;
    }
}

// atomic max on a float that may be negative (peak[t] initialised to -inf)
__device__ __forceinline__ void atomic_max_float(float *addr, float v)
{
    if(v >= 0.0f)
        atomicMax((int *)addr, __float_as_int(v));
    else
        atomicMin((unsigned int *)addr, __float_as_uint(v));
}

// dbfs, src/source.hpp:293-299 (libm-accurate form; used on rare paths and per-tick scalars)
__device__ __forceinline__ float dbfs(float mag, float db_min)
{
    return (mag > 0.0f) ? 20.0f * log10f(mag) : db_min;
}
// dbfs on the MUFU.LG2 path for the per-bin hot loops: 20 log10(m) = (20 log10 2) log2(m).  __log2f rescales
// subnormal inputs, so the reference's behaviour is kept over the whole float range (<= 2 ulp of log2).
__device__ __forceinline__ float dbfs_mufu(float mag, float db_min)
{
    return (mag > 0.0f) ? __log2f(mag) * 6.02059991327962390f : db_min;
}
// dbfs on the MUFU.LG2 path, two bins at a time (the N=2048, non-power-of-two and CTA-per-tick kernels).
// Magnitudes below FLT_MIN (digital silence, the far tail of an EMA decay: < -758.6 dBFS) report DB_MIN —
// the reference reports DB_MIN for exact zero and a value below DB_MIN for subnormals; this form clamps
// those to DB_MIN (dbfs_mufu keeps the exact behaviour).  See DESIGN.md §Parity.
__device__ __forceinline__ pk::c64 dbfs2(float m1, float m2, float db_min)
{
    constexpr float k = 6.02059991327962390f; // 20 log10(2)
    pk::c64 d = pk::mul(pk::make(lg2_approx_ftz(m1), lg2_approx_ftz(m2)), pk::make(k, k));
    // lg2.approx.ftz(x < FLT_MIN) = -inf and 20 log10(FLT_MIN) == DB_MIN, so the clamp is one max per bin
    float d1, d2;
    pk::split(d, d1, d2);
    return pk::make(fmaxf(d1, db_min), fmaxf(d2, db_min));
}

// ---- Stockham passes -------------------------------------------------------------------------------
// Pass with radix R, NS = product of previous radices.  v holds P = (M/R/TN)*R points: v[b*R + t].
template<int M, int TN, int R, int NS, bool FIRST>
struct Pass {
    static constexpr int BF = M / R;     // butterflies in this pass
    static constexpr int BPT = BF / TN;  // butterflies per thread
    static_assert(BPT >= 1 && BPT * TN == BF, "plan does not tile");

    template<int PP>
    static __device__ __forceinline__ void load_smem(float2 (&v)[PP], const float2 *buf, int tid)
    {
#pragma unroll
        for(int b = 0; b < BPT; ++b)
#pragma unroll
            for(int t = 0; t < R; ++t)
                v[b * R + t] = buf[phys(tid + b * TN + t * BF)];
    }

    // twiddle (for NS > 1), DFT-R, store in Stockham order
    template<int PP>
    static __device__ __forceinline__ void compute_store(float2 (&v)[PP], float2 *buf, const float2 *__restrict__ tw,
                                                         int tid)
    {
#pragma unroll
        for(int b = 0; b < BPT; ++b)
        {
            const int j = tid + b * TN;
            pk::c64 x[R]; // complex values as register pairs (see wf_fft.cuh)
#pragma unroll
            for(int t = 0; t < R; ++t)
                x[t] = pk::from(v[b * R + t]);
            if constexpr(NS > 1)
            {
                const int jm = j & (NS - 1);
                constexpr int STEP = M / (NS * R);
#pragma unroll
                for(int t = 1; t < R; ++t)
                    x[t] = pk::cmul(x[t], pk::from(__ldg(&tw[jm * t * STEP])));
            }
            pk::dft_bitrev<R>(x);
            const int base = (j / NS) * (NS * R) + (j & (NS - 1));
#pragma unroll
            for(int t = 0; t < R; ++t)
                buf[phys(base + t * NS)] = pk::to_float2(x[bitrev<R>(t)]);
        }
    }
};

template<int M, int TN, int NS, int... Rs>
struct LaterPasses;
template<int M, int TN, int NS>
struct LaterPasses<M, TN, NS> {
    template<int PP>
    static __device__ __forceinline__ void run(float2 (&)[PP], float2 *, const float2 *, int) {}
};
template<int M, int TN, int NS, int R, int... Rest>
struct LaterPasses<M, TN, NS, R, Rest...> {
    template<int PP>
    static __device__ __forceinline__ void run(float2 (&v)[PP], float2 *buf, const float2 *tw, int tid)
    {
        using PS = Pass<M, TN, R, NS, false>;
        group_sync<TN>(); // previous pass's stores are visible
        PS::load_smem(v, buf, tid);
        group_sync<TN>(); // everyone has read before anyone overwrites
        PS::compute_store(v, buf, tw, tid);
        LaterPasses<M, TN, NS * R, Rest...>::run(v, buf, tw, tid);
    }
};

template<int N, typename PlanType>
struct Fft;
template<int N, int TN_, int R0, int... Rest>
struct Fft<N, PlanT<TN_, R0, Rest...>> {
    static constexpr int M = N / 2;
    static constexpr int TN = TN_;
    static constexpr int P = M / TN;
    using P0 = Pass<M, TN, R0, 1, true>;

    // Issues the loads of one frame (as M complex points) into registers; no use of the values yet, so the loads
    // stay in flight across whatever the caller does next (software prefetch of the next tick).
    template<typename TS>
    static __device__ __forceinline__ void load_raw(float2 (&v)[P], const TS *frame, const KParams &p, int tid)
    {
        using PS = Pcm<TS>;
        if(p.aligned8)
        {
            const typename PS::Pair *f2 = reinterpret_cast<const typename PS::Pair *>(frame);
#pragma unroll
            for(int b = 0; b < P0::BPT; ++b)
#pragma unroll
                for(int t = 0; t < R0; ++t)
                    v[b * R0 + t] = PS::load2(f2 + (tid + b * TN + t * P0::BF));
        }
        else
        {
#pragma unroll
            for(int b = 0; b < P0::BPT; ++b)
#pragma unroll
                for(int t = 0; t < R0; ++t)
                {
                    const int n = tid + b * TN + t * P0::BF;
                    v[b * R0 + t] = make_float2(PS::load1(frame + 2 * n), PS::load1(frame + 2 * n + 1));
                }
        }
    }
    // Non-zero test (src/source_generic.cpp:63-76) and window multiply (:97-103) on a loaded frame.
    static __device__ __forceinline__ bool finish_load(float2 (&v)[P], const KParams &p, int tid)
    {
        bool nz = false;
#pragma unroll
        for(int i = 0; i < P; ++i)
            nz |= (v[i].x != 0.0f) | (v[i].y != 0.0f);
        if(p.window2 != nullptr)
        {
#pragma unroll
            for(int b = 0; b < P0::BPT; ++b)
#pragma unroll
                for(int t = 0; t < R0; ++t)
                {
                    const float2 w = __ldg(p.window2 + (tid + b * TN + t * P0::BF));
                    v[b * R0 + t].x *= w.x;
                    v[b * R0 + t].y *= w.y;
                }
        }
        return nz;
    }
    // Pulls a frame's cache lines into L2 (for plans whose register budget has no room for a register prefetch).
    template<typename TS>
    static __device__ __forceinline__ void prefetch_l2(const TS *frame, int tid)
    {
        constexpr int LINES = (N * Pcm<TS>::kBytes) / 128;
        for(int l = tid; l < LINES; l += TN)
            prefetch_l2_line(frame + l * (128 / Pcm<TS>::kBytes));
    }
    // Loads the frame (as M complex points), applies the window, reports whether any sample is nonzero.
    template<typename TS>
    static __device__ __forceinline__ bool load_frame(float2 (&v)[P], const TS *frame, const KParams &p, int tid)
    {
        load_raw(v, frame, p, tid);
        return finish_load(v, p, tid);
    }

    // Complex FFT of the M points in v; result X[k] (natural order) is left in buf[phys(k)].
    static __device__ __forceinline__ void run(float2 (&v)[P], float2 *buf, const float2 *tw, int tid)
    {
        group_sync<TN>(); // previous consumers of buf are done
        P0::compute_store(v, buf, tw, tid);
        LaterPasses<M, TN, R0, Rest...>::run(v, buf, tw, tid);
        group_sync<TN>(); // X visible to the whole group
    }
};

// The display stage's setup tables (interpolation indices / weights, bar bands, Gaussian): in global memory, read through
// the non-coherent path (LDG = true: the CTA-per-tick kernels), or copied once per CTA into shared memory by a persistent
// kernel (LDG = false: the warp-per-stream kernels, which evaluate ~n_points kernel sums per warp and tick).
struct DispTab {
    const float *interp_idx;
    const float *interp_w;
    const int *band_widths;
    const int *band_offsets;
    const float *gauss_w;
};
// copies the tables to `base` (16-byte aligned shared memory) with `nthreads` threads; the caller synchronises afterwards
__device__ __forceinline__ DispTab stage_display_tables(const KParams &p, float *base, int tid, int nthreads)
{
    const int n_idx = (p.n_sample > 0) ? p.n_sample : p.n_points;
    const int n_w = (p.interp_mode != 0) ? n_idx * p.taps : 0;
    const int n_g = p.filter ? p.gauss_size : 0, n_b = p.display_bar ? p.n_points : 0;
    float *t_w = base;
    float *t_idx = t_w + ((n_w + 3) & ~3);
    float *t_g = t_idx + n_idx;
    int *t_bw = reinterpret_cast<int *>(t_g + n_g);
    int *t_bo = t_bw + n_b;
    for(int i = tid; i < n_w; i += nthreads)
        t_w[i] = __ldg(p.interp_w + i);
    for(int i = tid; i < n_idx; i += nthreads)
        t_idx[i] = __ldg(p.interp_idx + i);
    for(int i = tid; i < n_g; i += nthreads)
        t_g[i] = __ldg(p.gauss_w + i);
    for(int i = tid; i < n_b; i += nthreads)
    {
        t_bw[i] = __ldg(p.band_widths + i);
        t_bo[i] = (p.band_offsets != nullptr) ? __ldg(p.band_offsets + i) : 0;
    }
    return DispTab{t_idx, t_w, t_bw, t_bo, t_g};
}
template<bool LDG, class T>
__device__ __forceinline__ T tab_ld(const T *q)
{
    if constexpr(LDG)
        return __ldg(q);
    else
        return *q;
}

// kernel_convolve, src/filter.hpp:160-169 (sequential mul+add, no contraction).  Away from the spectrum's edges the
// window is complete: all taps' weights (one or two 128-bit loads) and samples are fetched first, then accumulated in
// the reference's order — same rounding, no load latency inside the dependent chain.
template<int TAPS, bool LDG>
__device__ __forceinline__ float kernel_convolve_full(const float *db, const float *__restrict__ w)
{
    float wt[TAPS], x[TAPS];
#pragma unroll
    for(int q = 0; q < TAPS / 4; ++q)
    {
        const float4 w4 = tab_ld<LDG>(reinterpret_cast<const float4 *>(w) + q);
        wt[4 * q] = w4.x;
        wt[4 * q + 1] = w4.y;
        wt[4 * q + 2] = w4.z;
        wt[4 * q + 3] = w4.w;
    }
#pragma unroll
    for(int i = 0; i < TAPS; ++i)
        x[i] = db[i];
    float sum = 0.0f;
#pragma unroll
    for(int i = 0; i < TAPS; ++i)
        sum = __fadd_rn(sum, __fmul_rn(x[i], wt[i]));
    return sum;
}
template<bool LDG>
__device__ __forceinline__ float kernel_convolve(const float *db, int sz, const float *__restrict__ w, int radius, int index)
{
    const int start = (index - radius) + 1;
    const int stop = min(index + radius + 1, sz);
    if(start >= 0 && index + radius + 1 <= sz)
    {
        if(radius == 4)
            return kernel_convolve_full<8, LDG>(db + start, w); // Lanczos a = 4
        if(radius == 2)
            return kernel_convolve_full<4, LDG>(db + start, w); // Catmull-Rom
    }
    float sum = 0.0f;
    for(int i = max(start, 0); i < stop; ++i)
        sum = __fadd_rn(sum, __fmul_rn(db[i], tab_ld<LDG>(w + (i - start))));
    return sum;
}

// weighted_avg, src/filter.hpp:133-158
template<bool LDG>
__device__ __forceinline__ float weighted_avg(const KParams &p, const DispTab &tb, const float *samples, int n, int index)
{
    const int start = (index - p.gauss_radius) + 1;
    const int stop = index + p.gauss_radius;
    float sum = 0.0f;
    if((start < 0) || (stop > n))
    {
        const int loopstart = max(start, 0);
        const int loopstop = min(stop, n);
        float wsum = 0.0f;
        for(int i = loopstart; i < loopstop; ++i)
        {
            const float weight = tab_ld<LDG>(tb.gauss_w + (i - start));
            wsum = __fadd_rn(wsum, weight);
            sum = __fadd_rn(sum, __fmul_rn(samples[i], weight));
        }
        return __fdiv_rn(sum, wsum);
    }
    for(int i = start; i < stop; ++i)
        sum = __fadd_rn(sum, __fmul_rn(samples[i], tab_ld<LDG>(tb.gauss_w + (i - start))));
    return __fdiv_rn(sum, p.gauss_sum);
}

// std::lerp(float,float,float) as libstdc++ evaluates it (the plugin's lerp(), src/math_funcs.hpp:31-35), no contraction
__device__ __forceinline__ float std_lerp_dev(float a, float b, float t)
{
    if((a <= 0.0f && b >= 0.0f) || (a >= 0.0f && b <= 0.0f))
        return __fadd_rn(__fmul_rn(t, b), __fmul_rn(__fsub_rn(1.0f, t), a));
    if(t == 1.0f)
        return b;
    const float x = __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a)));
    return ((t > 1.0f) == (b > a)) ? (b < x ? x : b) : (b > x ? x : b);
}

// Render-time stages for one tick of one stream, from its dB spectrum `dbs` ([dch][B], shared or L2):
//   interpolation to display points (src/filter.hpp:182-211, src/source.cpp:1392-1394,1523-1532)
//   -> Gaussian smoothing (src/filter.hpp:133-180) -> out_points
//   -> dB -> pixel height (lerp/clamp), running (miny, minpos), frequency-axis mirroring
//      (src/source.cpp:1408-1424 curve, :1548-1565 bars) -> out_pixels / out_min
// `pts` is scratch for [2][dch][n_points] (+ [dch][n_sample]) floats: 4 * scratch_q floats per stream.  TN threads (one group) cooperate; SYNC() is the group barrier.
// A kernel sum with all TAPS taps.  Complete window: straight loads.  At the spectrum's edges the reference shortens the loop
// (src/filter.hpp:160-169); here the missing taps get weight 0 and a clamped address instead: adding x*0 = +-0 to the running
// sum leaves it unchanged (the skipped terms are leading or trailing, x is a finite dB value, the sum starts at +0), so the
// result is the same bit for bit without a divergent variable-length loop on the ~20 % of a log-frequency curve that sits
// on the first few bins.
template<int TAPS, bool LDG>
__device__ __forceinline__ float kernel_sum(const float *db, int sz, const float *__restrict__ w, int index)
{
    const int start = index - TAPS / 2 + 1;
    float wt[TAPS], x[TAPS];
#pragma unroll
    for(int q = 0; q < TAPS / 4; ++q)
    {
        const float4 w4 = tab_ld<LDG>(reinterpret_cast<const float4 *>(w) + q);
        wt[4 * q] = w4.x;
        wt[4 * q + 1] = w4.y;
        wt[4 * q + 2] = w4.z;
        wt[4 * q + 3] = w4.w;
    }
    if(start >= 0 && start + TAPS <= sz)
    {
#pragma unroll
        for(int i = 0; i < TAPS; ++i)
            x[i] = db[start + i];
    }
    else
    {
#pragma unroll
        for(int i = 0; i < TAPS; ++i)
        {
            const int j = start + i;
            const bool ok = (unsigned)j < (unsigned)sz;
            x[i] = db[ok ? j : 0];
            wt[i] = ok ? wt[i] : 0.0f;
        }
    }
    float sum = 0.0f;
#pragma unroll
    for(int i = 0; i < TAPS; ++i)
        sum = __fadd_rn(sum, __fmul_rn(x[i], wt[i]));
    return sum;
}

// value of sample point q of the interpolation tables; TAPS: 0 = nearest bin, 4 / 8 = Catmull-Rom / Lanczos kernel,
// -1 = any other radius (run-time loop)
template<bool LDG, int TAPS>
__device__ __forceinline__ float interp_at(const KParams &p, const DispTab &tb, const float *db, int B, int q)
{
    const int index = (int)tab_ld<LDG>(tb.interp_idx + q);
    if constexpr(TAPS == 0)
        return db[index];
    else if constexpr(TAPS > 0)
        return kernel_sum<TAPS, LDG>(db, B, tb.interp_w + (size_t)q * TAPS, index);
    else
        return kernel_convolve<LDG>(db, B, tb.interp_w + (size_t)q * p.taps, p.radius, index);
}

// Interpolation to display points (curve) or bars, with the mode tests outside the point loops.
template<int TN, bool LDG, int TAPS>
__device__ __forceinline__ void display_points(const KParams &p, const DispTab &tb, const float *dbs, float *raw, float *tmp, int B,
                                               int dch, size_t tick, int tid, bool active, bool need_smem)
{
    const int np = p.n_points;
    auto put = [&](int d, int i, float val) {
        if(need_smem)
            raw[d * np + i] = val;
        else if(active)
            stg_stream(p.out_points + (tick * dch + d) * np + i, val);
    };
    if(!p.display_bar)
    {
        for(int d = 0; d < dch; ++d)
            for(int i = tid; i < np; i += TN)
                put(d, i, interp_at<LDG, TAPS>(p, tb, dbs + d * B, B, i));
        return;
    }
    if constexpr(TAPS == 0)
    {
        // bars without a kernel: the mean of the band's bins (src/filter.hpp:195-211)
        for(int d = 0; d < dch; ++d)
            for(int i = tid; i < np; i += TN)
            {
                const int count = tab_ld<LDG>(tb.band_widths + i);
                const float *src = dbs + d * B + (int)tab_ld<LDG>(tb.interp_idx + i);
                float sum = 0.0f;
                for(int j = 0; j < count; ++j)
                    sum = __fadd_rn(sum, src[j]);
                put(d, i, __fdiv_rn(sum, (float)count));
            }
    }
    else
    {
        // Bars with an interpolation kernel: a bar is the mean of band_width kernel sums and the high-frequency bars are wide,
        // so one thread per bar would leave the group waiting for the widest bar.  Phase A evaluates every sample point of
        // every band in parallel; phase B adds them per bar in the reference's order.
        for(int d = 0; d < dch; ++d)
            for(int q = tid; q < p.n_sample; q += TN)
                tmp[d * p.n_sample + q] = interp_at<LDG, TAPS>(p, tb, dbs + d * B, B, q);
        group_sync<TN>();
        for(int d = 0; d < dch; ++d)
            for(int i = tid; i < np; i += TN)
            {
                const int count = tab_ld<LDG>(tb.band_widths + i);
                const float *src = tmp + d * p.n_sample + tab_ld<LDG>(tb.band_offsets + i);
                float sum = 0.0f;
                for(int j = 0; j < count; ++j)
                    sum = __fadd_rn(sum, src[j]);
                put(d, i, __fdiv_rn(sum, (float)count));
            }
    }
}

template<int TN, bool LDG>
__device__ __forceinline__ void display_stage_tab(const KParams &p, const DispTab &tb, const float *dbs, float *pts, float *tmp,
                                                  int B, int dch, size_t tick, int tid, bool active, float *red);
template<int TN>
__device__ __forceinline__ void display_stage(const KParams &p, const float *dbs, float *pts, int B, int dch, size_t tick,
                                              int tid, bool active, float *red)
{
    const DispTab tb{p.interp_idx, p.interp_w, p.band_widths, p.band_offsets, p.gauss_w};
    display_stage_tab<TN, true>(p, tb, dbs, pts, pts + 4 * p.n_points, B, dch, tick, tid, active, red);
}
// `tmp`: [dch][n_sample] floats (bars with an interpolation kernel), `pts`: [2][dch][n_points] floats (only touched when the
// Gaussian, pixel or minimum outputs are on), `red`: 2 * TN floats (pixel minimum only).
template<int TN, bool LDG>
__device__ __forceinline__ void display_stage_tab(const KParams &p, const DispTab &tb, const float *dbs, float *pts, float *tmp,
                                                  int B, int dch, size_t tick, int tid, bool active, float *red)
{
    const int np = p.n_points;
    const bool need_smem = p.filter || (p.out_pixels != nullptr) || (p.out_min != nullptr);
    float *raw = pts;                 // interpolated points
    float *fin = pts + dch * np;      // after the Gaussian (or alias of raw)
    if(p.interp_mode == 0 || (p.display_bar && p.n_sample <= 0))
        display_points<TN, LDG, 0>(p, tb, dbs, raw, tmp, B, dch, tick, tid, active, need_smem);
    else if(p.radius == 4 && p.taps == 8)
        display_points<TN, LDG, 8>(p, tb, dbs, raw, tmp, B, dch, tick, tid, active, need_smem);
    else if(p.radius == 2 && p.taps == 4)
        display_points<TN, LDG, 4>(p, tb, dbs, raw, tmp, B, dch, tick, tid, active, need_smem);
    else
        display_points<TN, LDG, -1>(p, tb, dbs, raw, tmp, B, dch, tick, tid, active, need_smem);
    if(!need_smem)
        return;
    group_sync<TN>();
    if(p.filter)
    {
        for(int d = 0; d < dch; ++d)
            for(int i = tid; i < np; i += TN)
                fin[d * np + i] = weighted_avg<LDG>(p, tb, raw + d * np, np, i);
        group_sync<TN>();
    }
    else
        fin = raw;
    if(p.out_points != nullptr && active)
        for(int i = tid; i < dch * np; i += TN)
            stg_stream(p.out_points + tick * dch * np + i, fin[i]);
    if(p.out_pixels == nullptr && p.out_min == nullptr)
        return;
    // dB -> pixels, in place; per-thread running minimum in (channel, index) order with strict '<'
    float my_min = INFINITY;
    int my_pos = 0x7fffffff;
    for(int d = 0; d < dch; ++d)
        for(int i = tid; i < np; i += TN)
        {
            const float c = fminf(fmaxf(__fsub_rn(p.ceiling_f, fin[d * np + i]), 0.0f), p.dbrange_f); // std::clamp
            const float val = std_lerp_dev(p.px_lo, p.px_hi, __fdiv_rn(c, p.dbrange_f));
            fin[d * np + i] = val;
            if(val < my_min)
            {
                my_min = val;
                my_pos = d * np + i;
            }
        }
    // group arg-min (ties -> earliest (channel, index), as the sequential scan of the reference does)
    red[2 * tid] = my_min;
    red[2 * tid + 1] = __int_as_float(my_pos);
    group_sync<TN>();
    if(tid == 0 && p.out_min != nullptr && active)
    {
        float miny = p.px_cpos;
        int minpos = 0;
        float best = INFINITY;
        int bpos = 0x7fffffff;
        for(int k = 0; k < TN; ++k)
        {
            const float v = red[2 * k];
            const int q = __float_as_int(red[2 * k + 1]);
            if(v < best || (v == best && q < bpos))
            {
                best = v;
                bpos = q;
            }
        }
        // sequential semantics: miny starts at cpos and only a strictly smaller value replaces it; minpos is the index
        // within its channel.  The reference resets nothing between channels, so a later channel wins only if smaller.
        if(best < miny)
        {
            miny = best;
            minpos = bpos % np;
        }
        p.out_min[tick * 2] = miny;
        p.out_min[tick * 2 + 1] = (float)minpos;
    }
    if(p.mirror)
    {
        group_sync<TN>();
        const int half = np / 2;
        // i > half takes the value at half - (i - half); sources (< half) are never overwritten
        for(int d = 0; d < dch; ++d)
            for(int i = half + 1 + tid; i < np; i += TN)
                fin[d * np + i] = fin[d * np + (half - (i - half))];
        group_sync<TN>();
    }
    if(p.out_pixels != nullptr && active)
        for(int i = tid; i < dch * np; i += TN)
            stg_stream(p.out_pixels + tick * dch * np + i, fin[i]);
    group_sync<TN>();
}

} // namespace wf
