// wf_fused.cuh — the fused per-frame spectrum pipeline as ONE sm_90a kernel:
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
#include "wf_kernels.cuh"

namespace wf {

template<int N, int CC, typename TS>
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

    const TS *pcm_s = Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride;
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
            const TS *frame = pcm_s + (size_t)c * p.channel_stride + (size_t)t * p.hop;
            if(!REGPF)
                F::load_raw(v, frame, p, tid);
            const bool nz = group_any<TN>(F::finish_load(v, p, tid));
            F::run(v, buf, p.tw, tid);
            {
                // next frame of this stream: the other channel of this tick, or channel 0 of the next tick
                const TS *next = (c + 1 < CC) ? frame + p.channel_stride
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
                float mag = sqrt_approx(pk::re(sq) + pk::im(sq)) * p.coef_half;
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

} // namespace wf
