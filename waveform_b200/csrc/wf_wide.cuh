// wf_wide.cuh — the fused spectrum pipeline for FEW streams x MANY ticks at large fft sizes (N >= 4096):
// a thread-block CLUSTER owns one stream and its R CTAs work on R consecutive ticks at once.
//
// Why: the EMA (src/source_generic.cpp:124-132) and the silence gate (:63-95) are recurrences over the ticks of
// a stream, so the one-group-per-stream kernel (wf_fused.cuh) can keep at most n_streams CTAs busy — BASELINE
// configs 4 and 5 have 128-256 streams per GPU, i.e. less than one small CTA per SM.  The FFT of a tick, however,
// does not depend on earlier ticks.  Per round of R ticks, CTA r of the cluster:
//   1. loads tick t0+r (prefetched during the previous round), windows it, runs the Stockham FFT and the real-FFT
//      split pass in its own shared memory -> linear magnitudes in registers;
//   2. scatters them through distributed shared memory so that CTA q receives bins [q*B/R, (q+1)*B/R) of all R
//      ticks (an all-to-all inside the cluster, ~B*4 bytes per CTA, no HBM traffic);
//   3. walks its B/R bins through the R ticks IN ORDER with the EMA state in registers — slope, EMA, channel mix,
//      dBFS, volume, roll-off exactly as wf_fused.cuh — and stores coalesced B/R-float row segments.
// HBM traffic stays the algorithmic minimum (each sample read once, each output written once); the recurrence is
// never parallelised, only distributed over bins, so results are bit-identical to the one-group kernel.
// The gate's all-bin reduction ("are last tick's outputs below floor-10 dB?") is evaluated lazily, only when a
// silent tick actually needs it, by one extra cluster barrier.  Display stages (interpolation, Gaussian, pixels)
// gather the finished dB spectrum of tick t0+r back into CTA r and reuse display_stage() of wf_kernels.cuh.
#pragma once
#include "wf_kernels.cuh"

namespace wf {
namespace wide {

// dynamic shared memory of one CTA: FFT exchange buffer (reused as the magnitude inbox) [+ dB gather + display scratch]
template<int N>
constexpr size_t smem_bytes(int dch, int n_points, bool display)
{
    size_t b = (size_t)Geo<N>::BUF * sizeof(float2);
    if(display)
        b += (size_t)dch * (N / 2) * sizeof(float) + (size_t)4 * n_points * sizeof(float);
    return b;
}

} // namespace wide

template<int N, int CC, int R, typename TS>
__global__ void __launch_bounds__(Geo<N>::TN, Geo<N>::MINB) stft_wide_kernel(const __grid_constant__ KParams p)
{
    using G = Geo<N>;
    using F = Fft<N, typename Plan<N>::type>;
    using P0 = typename F::P0;
    constexpr int M = G::M, B = G::M, TN = G::TN, P = G::P;
    constexpr int SLICE = B / R;   // bins owned by one CTA
    constexpr int SP = SLICE / TN; // bins owned by one thread
    static_assert(G::CTA == TN, "one frame per CTA");
    static_assert(SP >= 1 && SP * TN * R == B, "cluster size does not tile the bins");

    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);
    float *inbox = reinterpret_cast<float *>(smem_raw);              // [R][CC][SLICE] linear magnitudes (after barrier A)
    float *dbfull = reinterpret_cast<float *>(buf + G::BUF);        // [dch][B] dB spectrum of MY tick (display mode)
    float *pts = dbfull + (size_t)p.dch * B;                         // display scratch
    __shared__ float red_scratch[2 * TN];
    __shared__ unsigned nzf[R];        // per tick of the round: bit c = capture channel c has a non-zero sample
    __shared__ unsigned redf[2][R];    // gate reduction mailboxes (double-buffered)

    const int tid = threadIdx.x;
    const unsigned r = cluster_ctarank();
    const int s = blockIdx.x / R;
    const int T = p.n_frames;
    const int dch = p.dch, och = p.och;
    const bool stereo = p.stereo != 0;
    const bool want_points = (p.out_points != nullptr) || (p.out_pixels != nullptr) || (p.out_min != nullptr);
    const bool mirror_each_frame = (p.out_db == nullptr) && p.write_hold;

    const uint32_t inbox_sa = smem_u32(inbox);
    const uint32_t dbfull_sa = smem_u32(dbfull);

    // ---- my bins' EMA state -> registers ----
    float st[CC][SP];
    {
        const float *sp = p.state + (size_t)s * CC * B + r * SLICE;
#pragma unroll
        for(int c = 0; c < CC; ++c)
#pragma unroll
            for(int i = 0; i < SP; ++i)
                st[c][i] = sp[c * B + tid + i * TN];
    }
    const unsigned char fl = p.flags[s];
    bool last_silent = (fl & 1u) != 0;
    bool po0 = (fl & 2u) != 0, po1 = (fl & 4u) != 0; // previous tick's outputs all <= floor-10 (whole spectrum)
    bool po_valid = true;                            // po0/po1 are current; else the per-thread partials below are newer
    bool part0 = true, part1 = true;
    unsigned red_par = 0;

    const TS *pcm_s = Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride;
    float *hold_s = p.hold_db + (size_t)s * och * B;

    // cluster-wide AND of the per-thread partial flags of the last tick that produced outputs (rare path)
    auto ensure_po_valid = [&]() {
        if(po_valid)
            return;
        const int a0 = __syncthreads_and(part0 ? 1 : 0);
        const int a1 = __syncthreads_and(part1 ? 1 : 0);
        if(tid < R)
            st_cluster_u32(mapa(smem_u32(&redf[red_par][r]), (unsigned)tid), (unsigned)((a0 ? 1 : 0) | (a1 ? 2 : 0)));
        cluster_arrive();
        cluster_wait();
        unsigned all = 3u;
#pragma unroll
        for(int q = 0; q < R; ++q)
            all &= redf[red_par][q];
        po0 = (all & 1u) != 0;
        if(dch > 1)
            po1 = (all & 2u) != 0;
        red_par ^= 1u;
        po_valid = true;
    };

    float2 v[P];
    if((int)r < T)
        F::load_raw(v, pcm_s + (size_t)r * p.hop, p, tid); // channel 0 of my first tick

    // distributed shared memory may only be addressed once every CTA of the cluster has started executing
    cluster_arrive();
    cluster_wait();
    for(int t0 = 0; t0 < T; t0 += R)
    {
        const int nf = min(R, T - t0);
        const bool mine = (int)r < nf; // I hold tick t0 + r
        float magr[CC][P];
        unsigned nzbits = 0;

        // ---- phase 1: FFT + split pass + magnitude (+ slope) of my tick, src/source_generic.cpp:97-122 ----
        if(mine)
        {
#pragma unroll
            for(int c = 0; c < CC; ++c)
            {
                if(c > 0)
                    F::load_raw(v, pcm_s + (size_t)c * p.channel_stride + (size_t)(t0 + r) * p.hop, p, tid);
                const bool nz = group_any<TN>(F::finish_load(v, p, tid));
                nzbits |= nz ? (1u << c) : 0u;
                F::run(v, buf, p.tw, tid);
#pragma unroll
                for(int i = 0; i < P; ++i)
                {
                    const int k = tid + i * TN;
                    const pk::c64 a = pk::from(buf[phys(k)]);
                    const pk::c64 b = pk::conj(pk::from(buf[phys((M - k) & (M - 1))]));
                    const pk::c64 o = pk::mul_neg_i(pk::sub(a, b));
                    const pk::c64 y = pk::add(pk::add(a, b), pk::cmul(o, pk::from(__ldg(p.tw_post + k))));
                    const pk::c64 sq = pk::mul(y, y);
                    float mag = sqrt_approx(pk::re(sq) + pk::im(sq)) * p.coef_half;
                    if(p.slope != nullptr)
                        mag *= __ldg(p.slope + k);
                    magr[c][i] = mag;
                }
            }
        }
        __syncthreads(); // my FFT buffer is free: it becomes the inbox
        cluster_arrive(); // barrier A
        cluster_wait();

        // ---- phase 2: all-to-all — bins [q*SLICE, (q+1)*SLICE) of my tick go to CTA q ----
        if(mine)
        {
#pragma unroll
            for(int c = 0; c < CC; ++c)
#pragma unroll
                for(int i = 0; i < P; ++i)
                {
                    // bin k = tid + i*TN  ->  owner i / SP, offset tid + (i % SP) * TN   (SLICE is a multiple of TN)
                    const uint32_t dst = mapa(inbox_sa, (unsigned)(i / SP)) +
                                         (uint32_t)(((r * CC + c) * SLICE + tid + (i % SP) * TN) * sizeof(float));
                    st_cluster_f32(dst, magr[c][i]);
                }
            if(tid < R)
                st_cluster_u32(mapa(smem_u32(&nzf[r]), (unsigned)tid), nzbits);
        }
        cluster_arrive(); // barrier B
        // prefetch channel 0 of my next tick (the magnitudes have left the registers): in flight during phase 3
        if(t0 + R + (int)r < T)
            F::load_raw(v, pcm_s + (size_t)(t0 + R + r) * p.hop, p, tid);
        cluster_wait();

        // ---- phase 3: my bins through the round's ticks, in order ----
        for(int f = 0; f < nf; ++f)
        {
            const int t = t0 + f;
            const float2 gt = (p.g_tab != nullptr) ? __ldg(p.g_tab + t) : make_float2(p.g, p.g2); // gravity of this tick (src/source.hpp:301-312)
            const unsigned nzb = nzf[f];
            const bool skip_all = (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + t] != 0);
            bool proc[2] = {false, false};
            unsigned silent_channels = 0;
            const float *prev_db =
                (p.out_db != nullptr && t > 0) ? p.out_db + ((size_t)s * T + (t - 1)) * dch * B : hold_s;

#pragma unroll
            for(int c = 0; c < CC; ++c)
            {
                // gate, src/source_generic.cpp:63-95 (same state machine as wf_fused.cuh)
                bool do_proc = !skip_all;
                if(!skip_all)
                {
                    const bool silent = ((nzb >> c) & 1u) == 0;
                    if(!silent)
                        last_silent = false;
                    if(silent && p.gate)
                    {
                        if(last_silent)
                            do_proc = false;
                        else
                        {
                            bool outsilent;
                            if(!stereo && c == 1 && proc[0])
                                outsilent = false; // slot 0 holds channel 0's fresh linear magnitudes
                            else
                            {
                                ensure_po_valid();
                                outsilent = (stereo && c == 1) ? po1 : po0;
                            }
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
                // EMA, src/source_generic.cpp:124-132
#pragma unroll
                for(int i = 0; i < SP; ++i)
                {
                    float mag = inbox[(f * CC + c) * SLICE + tid + i * TN];
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

            // ---- outputs, src/source_generic.cpp:136-179 ----
            float vc = 0.0f;
            if(p.normalize)
            {
                const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + t] : 0.0f;
                vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
            }
            float *odb = (p.out_db != nullptr) ? p.out_db + ((size_t)s * T + t) * dch * B : nullptr;
            const uint32_t gather_sa = want_points ? mapa(dbfull_sa, (unsigned)f) : 0u;
            float peak = -INFINITY;
            bool outs0 = true, outs1 = true;
            for(int d = 0; d < dch; ++d)
            {
                bool outs = true;
#pragma unroll
                for(int i = 0; i < SP; ++i)
                {
                    const int k = r * SLICE + tid + i * TN;
                    float outv;
                    if(last_silent)
                        outv = prev_db[d * B + k]; // tick returned early (:138-139): m_decibels unchanged
                    else
                    {
                        float in;
                        if(CC == 2 && !stereo)
                        {
                            const float in0 = proc[0] ? st[0][i] : prev_db[k];
                            const float in1 = st[CC - 1][i];
                            in = (in0 + in1) * 0.5f; // :150-154
                        }
                        else
                        {
                            const int c = (CC == 2) ? d : 0;
                            in = proc[c] ? st[c][i] : prev_db[c * B + k];
                        }
                        outv = dbfs_mufu(in, p.db_min);
                        if(k >= 1)
                        {
                            if(p.normalize)
                                outv += vc; // :161-167
                            if(p.rolloff != nullptr)
                                outv = fmaxf(outv - __ldg(p.rolloff + k), p.db_min); // :169-179
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
                        st_cluster_f32(gather_sa + (uint32_t)((d * B + k) * sizeof(float)), outv);
                }
                if(d == 0)
                    outs0 = outs;
                else
                    outs1 = outs;
            }
            if(!last_silent && p.gate)
            {
                part0 = outs0;
                part1 = outs1;
                po_valid = false;
            }
            if(p.out_silent != nullptr && r == 0 && tid == 0)
                p.out_silent[(size_t)s * T + t] = last_silent ? 1 : 0;
            if(p.out_peak != nullptr)
            {
                const float gm = group_max<TN>(peak, red_scratch);
                if(tid == 0)
                    atomic_max_float(p.out_peak + t, gm);
            }
        }

        // ---- phase 4: render-time stages of my tick from the gathered dB spectrum ----
        if(want_points)
        {
            cluster_arrive(); // barrier C
            cluster_wait();
            if(mine)
                display_stage<TN>(p, dbfull, pts, B, dch, (size_t)s * T + t0 + r, tid, true, red_scratch);
        }
        __syncthreads(); // inbox reads are done before my next FFT overwrites the buffer
    }

    // ---- state back to the engine (my bins) ----
    ensure_po_valid();
    {
        float *sp = p.state + (size_t)s * CC * B + r * SLICE;
#pragma unroll
        for(int c = 0; c < CC; ++c)
#pragma unroll
            for(int i = 0; i < SP; ++i)
                sp[c * B + tid + i * TN] = st[c][i];
        if(p.write_hold && p.out_db != nullptr && T > 0)
        {
            const float *last = p.out_db + ((size_t)s * T + (T - 1)) * dch * B + r * SLICE;
            for(int d = 0; d < dch; ++d)
#pragma unroll
                for(int i = 0; i < SP; ++i)
                    hold_s[d * B + r * SLICE + tid + i * TN] = last[d * B + tid + i * TN];
        }
        if(CC == 2 && !stereo && p.write_hold)
        {
#pragma unroll
            for(int i = 0; i < SP; ++i)
                hold_s[B + r * SLICE + tid + i * TN] = st[1][i];
        }
        if(r == 0 && tid == 0)
            p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (po0 ? 2u : 0u) | (po1 ? 4u : 0u));
    }
    // no CTA may exit while a peer can still address its shared memory
    cluster_arrive();
    cluster_wait();
}

} // namespace wf
