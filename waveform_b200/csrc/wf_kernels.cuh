// wf_kernels.cuh — the fused per-frame spectrum pipeline as ONE sm_90a kernel:
//
//   PCM frame (HBM, read once) -> window multiply in the load prologue -> real-to-complex FFT as a
//   Stockham autosort FFT of the N/2 packed complex points (register radix-8/16/32 butterflies,
//   one padded shared-memory exchange per pass) -> split (hc2c) pass -> |X|·2/Σw -> slope ->
//   temporal EMA (state in registers across the frames of a stream) -> dBFS -> volume normalisation
//   -> roll-off -> coalesced store (HBM, written once) [-> log-frequency interpolation to curve /
//   bars -> Gaussian smoothing, from the dB spectrum kept in shared memory].
//
// Reference semantics restated here: WAVSourceGeneric::tick_spectrum src/source_generic.cpp:26-180,
// render-time interpolation src/source.cpp:1381-1406,1510-1546 + src/filter.hpp:133-211.
//
// Work decomposition: a GROUP of TN threads owns one stream (one WAVSource worth of state) and walks
// its n_frames ticks in order, because the EMA (src/source_generic.cpp:124-132) and the silence gate
// (:63-95) are recurrences over ticks.  Streams are independent -> grid = streams / groups-per-CTA.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "wf_fft.cuh"

namespace wf {

struct KParams {
    // input
    const float *pcm;
    long long stream_stride, channel_stride;
    int n_streams, n_frames, hop;
    int aligned8; // every frame start is 8-byte aligned -> float2 loads
    const float *input_rms;          // [n_streams][n_frames] or null
    const unsigned char *skip_mask;  // [n_streams][n_frames] or null
    // tables
    const float2 *window2; // window as float2[N/2] or null
    const float *window;   // same table, scalar view
    const float2 *tw;      // W_M^k
    const float2 *tw_post; // W_N^k, k < M
    const float *slope;    // or null
    const float *rolloff;  // or null
    // per-stream persistent state (already offset by first_stream)
    float *state;          // [streams][CC][B]   m_tsmooth_buf / last linear magnitude
    float *hold_db;        // [streams][OCH][B]  m_decibels as left by the last tick
    unsigned char *flags;  // [streams] bit0 last_silent, bit1/2 prev outputs of display slot 0/1 all <= floor-10
    // outputs
    float *out_db;             // [streams][frames][DCH][B] or null
    float *out_points;         // [streams][frames][DCH][n_points] or null
    unsigned char *out_silent; // [streams][frames] or null
    float *out_peak;           // [frames] or null (atomic max)
    // scalars
    float coef_half;  // (2 / window_sum) / 2
    float g, g2;      // gravity, 1 - gravity
    const float2 *g_tab; // optional [n_frames] (g, 1-g) per tick: TV-exponential smoothing with per-tick frame times
    int tsmooth;      // != 0: EMA enabled
    int fast_peaks;
    int stereo, och, dch;
    int gate;
    float floor_m10;  // (float)(floor - 10)
    float db_min;
    int normalize;
    float vol_target, max_gain;
    int write_hold;   // write final m_decibels mirror to hold_db at the end of the call
    int lazy_hold;    // N=2048 warp-per-stream kernel: leave the mirror implicit (flags bit 3) when it equals dbfs(state)
    int disp_bytes;   // warp-per-stream kernels with display outputs: extra shared memory per warp (dB row + display scratch)
    int disp_tab_bytes; // ... and per CTA (the display stage's setup tables)
    int split;        // N=2048 warp-per-stream kernel: cut an SM's frames into equal runs per warp (streams may change warps mid-call)
    // interpolation
    const float *interp_idx;
    const float *interp_w;
    const int *band_widths;
    const int *band_offsets;
    int n_points, taps, radius, display_bar, interp_mode;
    int n_sample;   // bars with a Lanczos / Catmull-Rom kernel: sample points of all bands (sum of band_widths), else 0
    int scratch_q;  // display scratch per stream = 4 * scratch_q floats (>= 4*n_points + dch*n_sample)
    const float *gauss_w;
    int gauss_radius, gauss_size;
    float gauss_sum;
    int filter;
    // display stage (dB -> pixels)
    float *out_pixels;     // [streams][frames][DCH][n_points] or null
    float *out_min;        // [streams][frames][2] or null
    float px_lo, px_hi;    // lerp endpoints: (0, cpos - channel_offset) for the curve, (border_top, border_bottom) for bars
    float px_cpos;         // initial miny
    float ceiling_f;       // (float)m_ceiling
    float dbrange_f;       // (float)(m_ceiling - m_floor)
    int mirror;
};

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

__device__ __forceinline__ float2 ldg_stream_f2(const float2 *p)
{
    float2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float ldg_stream_f1(const float *p)
{
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream(float *p, float v)
{
    asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
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
// sqrt on the MUFU path (subnormal-safe variant, max relative error 2^-23)
__device__ __forceinline__ float sqrt_mufu(float x)
{
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
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
    static __device__ __forceinline__ void load_raw(float2 (&v)[P], const float *frame, const KParams &p, int tid)
    {
        if(p.aligned8)
        {
            const float2 *f2 = reinterpret_cast<const float2 *>(frame);
#pragma unroll
            for(int b = 0; b < P0::BPT; ++b)
#pragma unroll
                for(int t = 0; t < R0; ++t)
                    v[b * R0 + t] = ldg_stream_f2(f2 + (tid + b * TN + t * P0::BF));
        }
        else
        {
#pragma unroll
            for(int b = 0; b < P0::BPT; ++b)
#pragma unroll
                for(int t = 0; t < R0; ++t)
                {
                    const int n = tid + b * TN + t * P0::BF;
                    v[b * R0 + t] = make_float2(ldg_stream_f1(frame + 2 * n), ldg_stream_f1(frame + 2 * n + 1));
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
    static __device__ __forceinline__ void prefetch_l2(const float *frame, int tid)
    {
        constexpr int LINES = (N * 4) / 128;
        for(int l = tid; l < LINES; l += TN)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(frame + l * 32));
    }
    // Loads the frame (as M complex points), applies the window, reports whether any sample is nonzero.
    static __device__ __forceinline__ bool load_frame(float2 (&v)[P], const float *frame, const KParams &p, int tid)
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
// floats of shared memory the tables take (weights padded to 16 bytes first, then indices, Gaussian, band widths, band offsets)
__host__ __device__ inline size_t display_table_floats(const KParams &p)
{
    const size_t n_idx = (p.n_sample > 0) ? (size_t)p.n_sample : (size_t)p.n_points;
    const size_t n_w = (p.interp_mode != 0) ? n_idx * (size_t)p.taps : 0;
    return ((n_w + 3) & ~(size_t)3) + n_idx + (p.filter ? (size_t)p.gauss_size : 0) + (p.display_bar ? 2 * (size_t)p.n_points : 0);
}
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

// ---- the fused kernel ------------------------------------------------------------------------------
template<int N, int CC>
__global__ void __launch_bounds__(Geo<N>::CTA, Geo<N>::MINB) stft_fused_kernel(const __grid_constant__ KParams p)
{
    using G = Geo<N>;
    using F = Fft<N, typename Plan<N>::type>;
    constexpr int M = G::M, B = G::M, TN = G::TN, P = G::P;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2 *smem = reinterpret_cast<float2 *>(smem_raw);
    const int grp = threadIdx.x / TN;
    const int tid = threadIdx.x % TN;
    float2 *buf = smem + (size_t)grp * G::BUF;
    float *dbs = reinterpret_cast<float *>(buf); // dB spectrum [dch][B] overlays the exchange buffer
    float *pts = reinterpret_cast<float *>(smem + (size_t)G::GROUPS * G::BUF) + (size_t)grp * 4 * p.scratch_q;
    __shared__ float red_scratch[2 * (G::CTA > 32 ? G::CTA : 32)];

    const int s_raw = blockIdx.x * G::GROUPS + grp;
    const bool active = s_raw < p.n_streams;
    const int s = active ? s_raw : (p.n_streams - 1);

    const int dch = p.dch, och = p.och;
    const bool stereo = p.stereo != 0;

    // ---- per-stream state -> registers ----
    float st[CC][P];
    {
        const float *sp = p.state + (size_t)s * CC * B;
#pragma unroll
        for(int c = 0; c < CC; ++c)
#pragma unroll
            for(int i = 0; i < P; ++i)
                st[c][i] = sp[c * B + tid + i * TN];
    }
    const unsigned char fl = p.flags[s];
    bool last_silent = (fl & 1u) != 0;
    bool prev_out_silent0 = (fl & 2u) != 0;
    bool prev_out_silent1 = (fl & 4u) != 0;

    const float *pcm_s = p.pcm + (size_t)s * p.stream_stride;
    float *hold_s = p.hold_db + (size_t)s * och * B;

    // Software pipelining of the PCM loads: plans with <= 16 points per thread keep the NEXT frame's samples in
    // registers across the epilogue; the others (no register room) pull the next frame into L2.
    constexpr bool REGPF = (P <= 16);
    float2 v[P];
    if(REGPF && p.n_frames > 0)
        F::load_raw(v, pcm_s, p, tid);

    for(int t = 0; t < p.n_frames; ++t)
    {
        const float2 gt = (p.g_tab != nullptr) ? __ldg(p.g_tab + t) : make_float2(p.g, p.g2); // gravity of this tick (src/source.hpp:301-312)
        const bool skip_all = (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * p.n_frames + t] != 0);
        bool proc[2] = {false, false};
        unsigned silent_channels = 0;

        // where the previous tick's m_decibels can be re-read (only on rare gate paths)
        const float *prev_db =
            (p.out_db != nullptr && t > 0) ? p.out_db + ((size_t)s * p.n_frames + (t - 1)) * dch * B : hold_s;
        const int prev_slot_stride = B;

#pragma unroll
        for(int c = 0; c < CC; ++c)
        {
            const float *frame = pcm_s + (size_t)c * p.channel_stride + (size_t)t * p.hop;
            if(!REGPF)
                F::load_raw(v, frame, p, tid);
            const bool nz = group_any<TN>(F::finish_load(v, p, tid));
            F::run(v, buf, p.tw, tid);
            {
                // next frame of this stream: the other channel of this tick, or channel 0 of the next tick
                const float *next = (c + 1 < CC) ? frame + p.channel_stride
                                                 : pcm_s + (size_t)(t + 1) * p.hop;
                if(c + 1 < CC || t + 1 < p.n_frames)
                {
                    if(REGPF)
                        F::load_raw(v, next, p, tid);
                    else
                        F::prefetch_l2(next, tid);
                }
            }

            // ---- gate, src/source_generic.cpp:63-95 ----
            bool do_proc = !skip_all;
            if(!skip_all)
            {
                const bool silent = !nz;
                if(!silent)
                    last_silent = false;
                if(silent && p.gate)
                {
                    if(last_silent)
                        do_proc = false;
                    else
                    {
                        // m_decibels[stereo ? channel : 0] all <= floor-10 ?  In mono-mix the second channel looks at
                        // slot 0, which holds channel 0's fresh LINEAR magnitudes (>= 0 > floor-10) if that was processed.
                        bool outsilent;
                        if(stereo)
                            outsilent = (c == 0) ? prev_out_silent0 : prev_out_silent1;
                        else
                            outsilent = (c == 1 && proc[0]) ? false : prev_out_silent0;
                        if(outsilent)
                        {
                            if(++silent_channels >= (unsigned)CC)
                                last_silent = true;
                            do_proc = false;
                        }
                    }
                }
            }
            proc[c] = do_proc;

            // ---- split pass + magnitude + slope + EMA, src/source_generic.cpp:110-135 ----
            // (computed unconditionally; committed to the state registers only if the channel is processed)
#pragma unroll
            for(int i = 0; i < P; ++i)
            {
                const int k = tid + i * TN;
                const pk::c64 a = pk::from(buf[phys(k)]);
                const pk::c64 b = pk::conj(pk::from(buf[phys((M - k) & (M - 1))]));
                const pk::c64 o = pk::mul_neg_i(pk::sub(a, b)); // -i (a - b)
                const pk::c64 y = pk::add(pk::add(a, b), pk::cmul(o, pk::from(__ldg(p.tw_post + k))));
                const pk::c64 sq = pk::mul(y, y);
                float mag = sqrt_mufu(pk::re(sq) + pk::im(sq)) * p.coef_half;
                if(p.slope != nullptr)
                    mag *= __ldg(p.slope + k);
                if(p.tsmooth)
                {
                    float oldval = st[c][i];
                    if(p.fast_peaks)
                        oldval = fmaxf(mag, oldval);
                    mag = __fadd_rn(__fmul_rn(gt.x, oldval), __fmul_rn(gt.y, mag));
                }
                if(do_proc)
                    st[c][i] = mag;
            }
        }

        // ---- outputs ----
        float vc = 0.0f;
        if(p.normalize)
        {
            const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * p.n_frames + t] : 0.0f;
            vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain); // src/source_generic.cpp:163
        }
        float *odb = (p.out_db != nullptr) ? p.out_db + ((size_t)s * p.n_frames + t) * dch * B : nullptr;
        const bool mirror_each_frame = (p.out_db == nullptr) && p.write_hold;
        const bool want_points = (p.out_points != nullptr) || (p.out_pixels != nullptr) || (p.out_min != nullptr);
        if(want_points)
            group_sync<TN>(); // split-pass reads of buf are done before dB overwrites it

        float peak = -INFINITY;
        bool outs0 = true, outs1 = true;
        for(int d = 0; d < dch; ++d)
        {
            bool outs = true;
#pragma unroll
            for(int i = 0; i < P; ++i)
            {
                const int k = tid + i * TN;
                float outv;
                if(last_silent)
                {
                    // tick returned early (src/source_generic.cpp:138-139): m_decibels unchanged
                    outv = prev_db[d * prev_slot_stride + k];
                }
                else
                {
                    float in;
                    if(CC == 2 && !stereo)
                    {
                        // 2 channels mixed to mono: dbfs((m0 + m1) * 0.5), src/source_generic.cpp:150-154
                        const float in0 = proc[0] ? st[0][i] : prev_db[k];
                        const float in1 = st[CC - 1][i];
                        in = (in0 + in1) * 0.5f;
                    }
                    else
                    {
                        // stereo with 2 channels: slot d <- channel d; mono source shown as stereo: slot 1 = copy of slot 0
                        const int c = (CC == 2) ? d : 0;
                        in = proc[c] ? st[c][i] : prev_db[c * prev_slot_stride + k];
                    }
                    outv = dbfs_mufu(in, p.db_min);
                    if(k >= 1)
                    {
                        if(p.normalize)
                            outv += vc; // src/source_generic.cpp:161-167
                        if(p.rolloff != nullptr)
                            outv = fmaxf(outv - __ldg(p.rolloff + k), p.db_min); // :169-179
                    }
                }
                outs &= !(outv > p.floor_m10);
                if(k >= 1)
                    peak = fmaxf(peak, outv);
                if(active)
                {
                    if(odb != nullptr)
                        stg_stream(odb + d * B + k, outv);
                    if(mirror_each_frame)
                        hold_s[d * B + k] = outv;
                }
                if(want_points)
                    dbs[d * B + k] = outv;
            }
            if(d == 0)
                outs0 = outs;
            else
                outs1 = outs;
        }
        if(!last_silent && p.gate)
        {
            prev_out_silent0 = group_all<TN>(outs0);
            if(dch > 1)
                prev_out_silent1 = group_all<TN>(outs1);
        }
        if(p.out_silent != nullptr && active && tid == 0)
            p.out_silent[(size_t)s * p.n_frames + t] = last_silent ? 1 : 0;
        if(p.out_peak != nullptr)
        {
            const float gm = group_max<TN>(peak, red_scratch);
            if(active && tid == 0)
                atomic_max_float(p.out_peak + t, gm);
        }

        // ---- render-time stages from the dB spectrum in shared memory ----
        if(want_points)
        {
            group_sync<TN>();
            display_stage<TN>(p, dbs, pts, B, dch, (size_t)s * p.n_frames + t, tid, active, red_scratch + grp * 2 * TN);
        }
    }

    // ---- state back to the engine ----
    if(active)
    {
        float *sp = p.state + (size_t)s * CC * B;
#pragma unroll
        for(int c = 0; c < CC; ++c)
#pragma unroll
            for(int i = 0; i < P; ++i)
                sp[c * B + tid + i * TN] = st[c][i];
        if(p.write_hold && p.out_db != nullptr && p.n_frames > 0)
        {
            // m_decibels mirror := outputs of the last tick (slot 1 of a mono mix keeps linear channel-1 magnitudes)
            const float *last = p.out_db + ((size_t)s * p.n_frames + (p.n_frames - 1)) * dch * B;
            for(int d = 0; d < dch; ++d)
#pragma unroll
                for(int i = 0; i < P; ++i)
                    hold_s[d * B + tid + i * TN] = last[d * B + tid + i * TN];
        }
        if(CC == 2 && !stereo && p.write_hold)
        {
#pragma unroll
            for(int i = 0; i < P; ++i)
                hold_s[B + tid + i * TN] = st[1][i];
        }
        if(tid == 0)
            p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (prev_out_silent0 ? 2u : 0u) | (prev_out_silent1 ? 4u : 0u));
    }
}

// Streams whose m_decibels mirror was left implicit by stft2048_fast_kernel (flags bit 3: mirror == dbfs(state), one
// capture channel, one display channel) get it written out here, with the same MUFU.LG2 arithmetic the kernel used for
// the outputs.  Run by the engine before anything else reads hold_db (other kernels, wf_get_state / wf_set_state).
static __global__ void materialize_hold_kernel(const float *state, float *hold_db, unsigned char *flags, int n_streams, int B,
                                               int och, float db_min)
{
    for(int s = blockIdx.x; s < n_streams; s += gridDim.x)
    {
        const unsigned char fl = flags[s];
        if(!(fl & 8u))
            continue;
        for(int k = threadIdx.x; k < B; k += blockDim.x)
        {
            float l;
            asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(state[(size_t)s * B + k]));
            hold_db[(size_t)s * och * B + k] = fmaxf(l * 6.02059991327962390f, db_min);
        }
        __syncthreads();
        if(threadIdx.x == 0)
            flags[s] = (unsigned char)(fl & ~8u);
    }
}

// Timeout / hidden branch of tick_spectrum (src/source_generic.cpp:36-48) for streams [0, n_streams): a stream that is
// already m_last_silent returns early there and keeps its buffers; the others get m_tsmooth_buf := 0, the DISPLAY rows of
// m_decibels := DB_MIN (slot 1 of a 2ch->mono mix keeps its last linear magnitudes, :43-45) and m_last_silent := true.
static __global__ void spectrum_reset_kernel(float *state, float *hold_db, unsigned char *flags, int n_streams, int ccB, int ochB,
                                             int dchB, float db_min, unsigned char new_flags)
{
    for(int s = blockIdx.x; s < n_streams; s += gridDim.x)
    {
        if(flags[s] & 1u)
            continue;
        for(int i = threadIdx.x; i < ccB; i += blockDim.x)
            state[(size_t)s * ccB + i] = 0.0f;
        for(int i = threadIdx.x; i < dchB; i += blockDim.x)
            hold_db[(size_t)s * ochB + i] = db_min;
        __syncthreads();
        if(threadIdx.x == 0)
            flags[s] = new_flags;
    }
}

// peak normalisation pass: out[row][k] += gain[t] for k >= 1 (row = (stream, frame, channel))
static __global__ void peak_normalize_kernel(float *data, int n_streams, int n_frames, int rows_per_frame, int row_len,
                                      const float *peak, float target_db, float max_gain)
{
    const long long rows = (long long)n_streams * n_frames * rows_per_frame;
    for(long long r = blockIdx.x; r < rows; r += gridDim.x)
    {
        const int t = (int)((r / rows_per_frame) % n_frames);
        const float gain = fminf(target_db - peak[t], max_gain);
        float *row = data + r * row_len;
        for(int k = 1 + threadIdx.x; k < row_len; k += blockDim.x)
            row[k] += gain;
    }
}

static __global__ void fill_kernel(float *p, long long n, float v)
{
    for(long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        p[i] = v;
}

} // namespace wf
