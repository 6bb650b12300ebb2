// wf_anyn.cuh — the same fused pipeline for ANY fft_size the plugin can produce (multiples of 16 that are not
// powers of two: the slider's 64-sample steps, and the automatic size sr/fps & -16, e.g. 800 at 48 kHz / 60 fps;
// src/source.cpp:349,562-565,1161-1167).  SURVEY.md §8(f) rank 1.
//
// The N/2-point complex FFT is a run-time mixed-radix Stockham FFT in shared memory: one pass per factor of N/2
// (factors of two grouped up to 16, odd primes taken as they are), every output element formed directly as
//     out[o] = sum_u in[j + u*M/r] * W_M^(u*step),   step = low*M/(Ns*r) + t*M/r   (pass twiddle x radix-r DFT matrix)
// — O(M * sum(r)) multiply-adds per frame instead of hand-unrolled butterflies: this path favours generality over
// speed (the power-of-two kernels are the fast ones).  Everything after the FFT (split pass, magnitude, slope, EMA,
// gate, dBFS, volume, roll-off, interpolation, Gaussian) restates the same reference lines as wf_fused.cuh.
#pragma once
#include "wf_anyn.hpp"
#include "wf_kernels.cuh"

namespace wf {

template<int CC, typename TS>
__global__ void __launch_bounds__(kAnyThreads) stft_anyn_kernel(const __grid_constant__ KParams p,
                                                                  const __grid_constant__ AnyPlan plan)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int M = plan.M, B = plan.M;
    float2 *bufA = (plan.scratch != nullptr) ? plan.scratch + (size_t)blockIdx.x * 2 * M : reinterpret_cast<float2 *>(smem_raw);
    float2 *bufB = bufA + M;
    // [dch][n_points] intermediate of the Gaussian (only when filtering display points)
    float *pts = (plan.scratch != nullptr) ? reinterpret_cast<float *>(smem_raw) : reinterpret_cast<float *>(bufB + M);
    __shared__ float red_scratch[2 * kAnyThreads];
    const int tid = threadIdx.x;
    const int dch = p.dch, och = p.och;
    const bool stereo = p.stereo != 0;
    const int T = p.n_frames;

    for(int s = blockIdx.x; s < p.n_streams; s += gridDim.x)
    {

    float *state_s = p.state + (size_t)s * CC * B;
    float *hold_s = p.hold_db + (size_t)s * och * B;
    const unsigned char fl = p.flags[s];
    bool last_silent = (fl & 1u) != 0;
    bool prev_out_silent0 = (fl & 2u) != 0;
    bool prev_out_silent1 = (fl & 4u) != 0;
    const TS *pcm_s = Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride;

    for(int t = 0; t < T; ++t)
    {
        const float2 gt = (p.g_tab != nullptr) ? __ldg(p.g_tab + t) : make_float2(p.g, p.g2); // gravity of this tick (src/source.hpp:301-312)
        const bool skip_all = (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + t] != 0);
        bool proc[2] = {false, false};
        unsigned silent_channels = 0;
        const float *prev_db = (p.out_db != nullptr && t > 0) ? p.out_db + ((size_t)s * T + (t - 1)) * dch * B : hold_s;

        for(int c = 0; c < CC; ++c)
        {
            // ---- frame + window -> bufA (packed as N/2 complex points) ----
            const TS *frame = pcm_s + (size_t)c * p.channel_stride + (size_t)t * p.hop;
            bool nzl = false;
            __syncthreads(); // previous users of the buffers are done
            for(int n = tid; n < M; n += kAnyThreads)
            {
                float2 z = make_float2(Pcm<TS>::load1(frame + 2 * n), Pcm<TS>::load1(frame + 2 * n + 1));
                nzl |= (z.x != 0.0f) | (z.y != 0.0f);
                if(p.window != nullptr)
                {
                    z.x *= __ldg(p.window + 2 * n);
                    z.y *= __ldg(p.window + 2 * n + 1);
                }
                bufA[n] = z;
            }
            const bool nz = __syncthreads_or(nzl) != 0;

            // ---- mixed-radix Stockham passes ----
            float2 *src = bufA, *dst = bufB;
            int Ns = 1;
            for(int ps = 0; ps < plan.n_pass; ++ps)
            {
                const int r = plan.radix[ps];
                const int BF = M / r;
                const int unit = M / (Ns * r);
                for(int o = tid; o < M; o += kAnyThreads)
                {
                    const int low = o % Ns;
                    const int tt = (o / Ns) % r;
                    const int high = o / (Ns * r);
                    const int j = high * Ns + low;
                    int step = low * unit + tt * BF;
                    step -= (step >= M) ? M : 0;
                    // The r terms are summed in three levels: blocks of 32 terms, blocks of 32 block sums, then those in
                    // order.  One running float32 sum over a large prime radix (1021, 4093 at the plugin's largest
                    // sizes) grows its rounding error with r: 2.1e-5 normwise at N = 65488 on an H100 (DESIGN §2).
                    // Radices up to 32 are one block: the same operations as a single running sum.
                    float2 acc = src[j], mid = make_float2(0.0f, 0.0f), tot = make_float2(0.0f, 0.0f);
                    int e = 0;
                    for(int u = 1; u < r; ++u)
                    {
                        e += step;
                        e -= (e >= M) ? M : 0;
                        if((u & 31) == 0)
                        {
                            mid = cadd(mid, acc);
                            acc = make_float2(0.0f, 0.0f);
                            if((u & 1023) == 0)
                            {
                                tot = cadd(tot, mid);
                                mid = make_float2(0.0f, 0.0f);
                            }
                        }
                        acc = cadd(acc, cmul(src[j + u * BF], __ldg(p.tw + e)));
                    }
                    dst[o] = (r > 32) ? cadd(tot, cadd(mid, acc)) : acc;
                }
                __syncthreads();
                float2 *tmp = src;
                src = dst;
                dst = tmp;
                Ns *= r;
            }
            const float2 *X = src;

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

            // ---- split pass + magnitude + slope + EMA (state lives in global memory / L2 on this path) ----
            if(do_proc)
            {
                float *st = state_s + (size_t)c * B;
                for(int k = tid; k < B; k += kAnyThreads)
                {
                    const float2 a = X[k];
                    float2 b = X[(k == 0) ? 0 : (M - k)];
                    b.y = -b.y;
                    const float2 sum = cadd(a, b);
                    const float2 dif = csub(a, b);
                    const float2 o = make_float2(dif.y, -dif.x);
                    const float2 y = cadd(sum, cmul(o, __ldg(p.tw_post + k)));
                    float mag = sqrt_approx(fmaf(y.x, y.x, y.y * y.y)) * p.coef_half;
                    if(p.slope != nullptr)
                        mag *= __ldg(p.slope + k);
                    if(p.tsmooth)
                    {
                        float oldval = st[k];
                        if(p.fast_peaks)
                            oldval = fmaxf(mag, oldval);
                        mag = __fadd_rn(__fmul_rn(gt.x, oldval), __fmul_rn(gt.y, mag));
                    }
                    st[k] = mag;
                }
            }
        }
        __syncthreads(); // state writes visible to the output stage; FFT buffers free

        // ---- outputs ----
        float vc = 0.0f;
        if(p.normalize)
        {
            const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + t] : 0.0f;
            vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
        }
        float *odb = (p.out_db != nullptr) ? p.out_db + ((size_t)s * T + t) * dch * B : nullptr;
        const bool mirror_each_frame = (p.out_db == nullptr) && p.write_hold;
        const bool want_points = (p.out_points != nullptr) || (p.out_pixels != nullptr) || (p.out_min != nullptr);
        float *dbs = reinterpret_cast<float *>(bufA); // dB spectrum [dch][B] for the display stage (2B floats fit)
        float peak = -INFINITY;
        bool outs0 = true, outs1 = true;
        for(int d = 0; d < dch; ++d)
        {
            bool outs = true;
            for(int k = tid; k < B; k += kAnyThreads)
            {
                float outv;
                if(last_silent)
                    outv = prev_db[d * B + k];
                else
                {
                    float in;
                    if(CC == 2 && !stereo)
                    {
                        const float in0 = proc[0] ? state_s[k] : prev_db[k];
                        in = (in0 + state_s[B + k]) * 0.5f;
                    }
                    else
                    {
                        const int c = (CC == 2) ? d : 0;
                        in = proc[c] ? state_s[(size_t)c * B + k] : prev_db[c * B + k];
                    }
                    outv = dbfs_mufu(in, p.db_min);
                    if(k >= 1)
                    {
                        if(p.normalize)
                            outv += vc;
                        if(p.rolloff != nullptr)
                            outv = fmaxf(outv - __ldg(p.rolloff + k), p.db_min);
                    }
                }
                outs &= !(outv > p.floor_m10);
                if(k >= 1)
                    peak = fmaxf(peak, outv);
                if(odb != nullptr)
                    stg_stream(odb + d * B + k, outv);
                if(mirror_each_frame)
                    hold_s[d * B + k] = outv;
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
            prev_out_silent0 = __syncthreads_and(outs0) != 0;
            if(dch > 1)
                prev_out_silent1 = __syncthreads_and(outs1) != 0;
        }
        if(p.out_silent != nullptr && tid == 0)
            p.out_silent[(size_t)s * T + t] = last_silent ? 1 : 0;
        if(p.out_peak != nullptr)
        {
            const float gm = group_max<kAnyThreads>(peak, red_scratch);
            if(tid == 0)
                atomic_max_float(p.out_peak + t, gm);
        }
        if(want_points)
        {
            __syncthreads();
            display_stage<kAnyThreads>(p, dbs, pts, B, dch, (size_t)s * T + t, tid, true, red_scratch);
        }
    }

    // ---- m_decibels mirror + flags back to the engine (state is already in place) ----
    __syncthreads();
    if(p.write_hold && p.out_db != nullptr && T > 0)
    {
        const float *last = p.out_db + ((size_t)s * T + (T - 1)) * dch * B;
        for(int i = tid; i < dch * B; i += kAnyThreads)
            hold_s[i] = last[i];
    }
    if(CC == 2 && !stereo && p.write_hold)
        for(int k = tid; k < B; k += kAnyThreads)
            hold_s[B + k] = state_s[B + k];
    if(tid == 0)
        p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (prev_out_silent0 ? 2u : 0u) | (prev_out_silent1 ? 4u : 0u));
    __syncthreads();
    } // streams
}

} // namespace wf
