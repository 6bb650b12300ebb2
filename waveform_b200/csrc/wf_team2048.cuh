// wf_team2048.cuh — N = 2048, one capture channel, spectrum output, FEW streams x MANY ticks (SURVEY §8(d) C3 "256 x 256").
//
// The warp-per-stream kernel (wf_fast2048.cuh) needs ~2100 streams to fill 132 SMs x 16 warps.  With fewer streams the only
// sequential part of a stream is the EMA / gate recurrence over ticks — the FFT of a tick is not.  Here a TEAM of W warps
// (W = 4, 8, 16; 16/W teams per CTA, one CTA per SM) owns a stream and works on W consecutive ticks at once:
//
//   phase 1 (per warp = per tick): TMA-staged frame -> window -> packed 1024-point complex FFT (two radix-32 register
//            passes, one padded shared-memory transpose) -> split pass on bin pairs -> |X| (-> slope): exactly the
//            arithmetic of wf_fast2048.cuh; the linear magnitudes of the tick go to the warp's 4 KB slot in shared memory
//            in natural bin order.
//   team barrier (bar.sync on a named barrier, W*32 threads)
//   phase 2 (per warp = per bin slice): warp j owns bins [j*1024/W, (j+1)*1024/W), lane l owns 32/W consecutive ones; it
//            walks the W ticks IN ORDER with the EMA state in registers: EMA -> dBFS (MUFU.LG2) -> (volume, roll-off) ->
//            one 128-bit coalesced store per 4 bins.  The gate's all-bins test ("outputs already <= floor-10 dB") is a
//            per-lane running flag, reduced over the team only when a silent tick actually needs it (two extra barriers).
//   team barrier (the magnitude slots are free again)
//
// Recurrences are distributed over bins, never reassociated: results are bit-identical to wf_fast2048.cuh.
// Semantics: src/source_generic.cpp:26-180 as restated there.
#pragma once
#include "wf_fast2048.cuh"

namespace wf {

namespace team {
constexpr int kCtlBytes = 64;  // per team: nz[16] | outs[16] (bytes)
constexpr int kWarps = 16;
constexpr int smem_bytes() { return fast::kTableBytes + kWarps * fast::kWarpBytes + kWarps * kCtlBytes; }

__device__ __forceinline__ void bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
} // namespace team

template<int W, bool EXTRA>
__global__ void __launch_bounds__(team::kWarps * 32, 1) stft2048_team_kernel(const __grid_constant__ KParams p)
{
    using namespace fast;
    constexpr int TPC = team::kWarps / W; // teams per CTA
    constexpr int BW = kM / W;            // bins per warp in phase 2
    constexpr int BPL = BW / 32;          // bins per lane: 2, 4, 8, 16
    constexpr int VEC = (BPL >= 4) ? 4 : 2;
    constexpr int B = kM;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2 *s_win = reinterpret_cast<float2 *>(smem_raw);
    float2 *s_twA = s_win + 1024; // [k2][n1] = W_1024^(k2*n1)
    float2 *s_twP = s_twA + 1024; // [q][lane] = W_2048^(lane + 32 q), q < 16
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int tm = warp / W; // team within the CTA
    const int wi = warp % W; // warp within the team = tick within a round (phase 1) = bin slice (phase 2)
    unsigned char *warps_base = reinterpret_cast<unsigned char *>(s_twP + 512);
    unsigned char *wbase = warps_base + warp * kWarpBytes;
    float2 *buf = reinterpret_cast<float2 *>(wbase);
    float *mymag = reinterpret_cast<float *>(wbase + kWarpBufBytes); // this warp's tick: linear magnitudes [1024]
    uint64_t *mbar = reinterpret_cast<uint64_t *>(wbase + kWarpBufBytes + kStateBytes);
    unsigned char *ctl = warps_base + team::kWarps * kWarpBytes + tm * team::kCtlBytes;
    volatile unsigned char *ctl_nz = ctl;         // [W] frame of tick t0+i has a non-zero sample
    volatile unsigned char *ctl_outs = ctl + 16;  // [W] per-warp partial of the gate's all-bins test
    const int bar_id = 1 + tm;

    for(int i = threadIdx.x; i < 1024; i += blockDim.x)
    {
        const float2 w = (p.window2 != nullptr) ? __ldg(p.window2 + i) : make_float2(1.0f, 1.0f);
        s_win[i] = make_float2(w.x * p.coef_half, w.y * p.coef_half);
        s_twA[i] = __ldg(p.tw + (((i >> 5) * (i & 31)) & 1023));
        if(i < 512)
            s_twP[i] = __ldg(p.tw_post + i);
    }
    if(lane == 0)
    {
        mbar_init(mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // streams are dealt round-robin to CTAs first, then to the CTA's teams: stream of (cta c, team tm, i) = c + G*(tm + TPC*i)
    const int S = p.n_streams, T = p.n_frames;
    const int G = gridDim.x;
    const int n_local = (S > (int)blockIdx.x) ? (S - (int)blockIdx.x + G - 1) / G : 0;
    uint32_t phase = 0;
    const bool tsm = p.tsmooth != 0, gate = p.gate != 0;

    // phase-1 bin pairs of this lane (as in wf_fast2048.cuh)
    const int jp = (32 - lane) & 31;
    const int kb = jp + (lane == 0 ? 32 : 0);
    const int k2_q0 = (lane == 0) ? 512 : (kb + 992);
    // phase-2 bins of this lane
    const int b0 = wi * BW + lane * BPL;

    // first frame of this warp: tick wi of the team's first stream
    if(tm < n_local && wi < T && lane == 0)
    {
        mbar_expect_tx(mbar, kN * 4);
        tma_load_1d(buf, p.pcm + (size_t)(blockIdx.x + tm * G) * p.stream_stride + (size_t)wi * p.hop, kN * 4, mbar);
    }

    for(int li = tm; li < n_local; li += TPC)
    {
        const int s = (int)blockIdx.x + li * G;
        const bool have_next_stream = (li + TPC) < n_local;
        const float *pcm_s = p.pcm + (size_t)s * p.stream_stride;
        float *hold_s = p.hold_db + (size_t)s * B;
        float *state_s = p.state + (size_t)s * B;

        // ---- per-stream state: this lane's bins -> registers ----
        float st[BPL];
#pragma unroll
        for(int j = 0; j < BPL; j += VEC)
        {
            if constexpr(VEC == 4)
            {
                const float4 x = *reinterpret_cast<const float4 *>(state_s + b0 + j);
                st[j] = x.x, st[j + 1] = x.y, st[j + 2] = x.z, st[j + 3] = x.w;
            }
            else
            {
                const float2 x = *reinterpret_cast<const float2 *>(state_s + b0 + j);
                st[j] = x.x, st[j + 1] = x.y;
            }
        }
        const unsigned char fl = p.flags[s];
        bool last_silent = (fl & 1u) != 0;
        bool pos = (fl & 2u) != 0;   // prev_out_silent: all outputs of the last producing tick <= floor-10 dB ...
        bool pos_valid = true;       // ... evaluated lazily from the per-lane flags when false
        bool outs_lane = true;
        const bool hold_lazy = (fl & 8u) != 0;
        bool last_from_state = false;

        // team-wide AND of the per-lane flags (rare: only when a silent tick needs the answer, and once at the stream's end)
        auto team_all = [&](bool v) -> bool {
            const bool wv = __all_sync(0xffffffffu, v);
            if(lane == 0)
                ctl_outs[wi] = wv ? 1 : 0;
            team::bar_sync(bar_id, W * 32);
            bool r = true;
#pragma unroll
            for(int i = 0; i < W; ++i)
                r &= ctl_outs[i] != 0;
            team::bar_sync(bar_id, W * 32);
            return r;
        };

        for(int t0 = 0; t0 < T; t0 += W)
        {
            // =================== phase 1: this warp transforms tick t0 + wi ===================
            const int t = t0 + wi;
            if(t < T)
            {
                mbar_wait(mbar, phase);
                phase ^= 1u;
                pk::c64 v[32];
                unsigned long long nzbits = 0;
                const pk::c64 *buf64 = reinterpret_cast<const pk::c64 *>(buf);
                const pk::c64 *win64 = reinterpret_cast<const pk::c64 *>(s_win);
#pragma unroll
                for(int pidx = 0; pidx < 32; ++pidx)
                {
                    v[pidx] = buf64[lane + 32 * pidx];
                    nzbits |= v[pidx];
                }
#pragma unroll
                for(int pidx = 0; pidx < 32; ++pidx)
                    v[pidx] = pk::mul(v[pidx], win64[lane + 32 * pidx]);
                const bool nz = __any_sync(0xffffffffu, (nzbits & 0x7fffffff7fffffffull) != 0ull);
#pragma unroll
                for(int pass = 0; pass < 2; ++pass)
                {
                    pk::dft_bitrev<32>(v);
                    if(pass == 0)
                    {
                        __syncwarp();
#pragma unroll
                        for(int k2 = 0; k2 < 32; ++k2)
                        {
                            pk::c64 a = v[bitrev<32>(k2)];
                            if(k2 > 0)
                                a = pk::cmul(a, reinterpret_cast<const pk::c64 *>(s_twA)[k2 * 32 + lane]);
                            reinterpret_cast<pk::c64 *>(buf)[lane * 33 + k2] = a;
                        }
                        __syncwarp();
#pragma unroll
                        for(int n1 = 0; n1 < 32; ++n1)
                            v[n1] = buf64[n1 * 33 + lane];
                        __syncwarp();
                        // next frame of this warp: tick t + W of this stream, else tick wi of the team's next stream
                        const float *next = nullptr;
                        if(t + W < T)
                            next = pcm_s + (size_t)(t + W) * p.hop;
                        else if(have_next_stream)
                            next = p.pcm + (size_t)(s + TPC * G) * p.stream_stride + (size_t)wi * p.hop;
                        if(lane == 0 && next != nullptr)
                        {
                            fence_proxy_async();
                            mbar_expect_tx(mbar, kN * 4);
                            tma_load_1d(buf, next, kN * 4, mbar);
                        }
                    }
                }
                // split pass on pairs -> |X| (-> slope) -> this warp's magnitude slot, natural bin order
#pragma unroll
                for(int q = 0; q < 16; ++q)
                {
                    const int k1 = lane + 32 * q;
                    const int k2 = (q == 0) ? k2_q0 : (kb + 32 * (31 - q));
                    const pk::c64 a = v[bitrev<32>(q)];
                    unsigned long long bp = __shfl_sync(0xffffffffu, v[bitrev<32>(31 - q)], jp);
                    if(lane == 0)
                        bp = v[bitrev<32>((32 - q) & 31)];
                    const pk::c64 b = pk::conj(bp);
                    const pk::c64 sum = pk::add(a, b);
                    const pk::c64 o = pk::mul_neg_i(pk::sub(a, b));
                    const pk::c64 wo = pk::cmul(o, reinterpret_cast<const pk::c64 *>(s_twP)[q * 32 + lane]);
                    const pk::c64 y1 = pk::add(sum, wo);
                    const pk::c64 y2 = pk::sub(sum, wo);
                    const pk::c64 s1 = pk::mul(y1, y1), s2 = pk::mul(y2, y2);
                    float p1 = pk::re(s1) + pk::im(s1);
                    float p2 = pk::re(s2) + pk::im(s2);
                    if(q == 0)
                    {
                        const pk::c64 x512 = v[bitrev<32>(16)];
                        const pk::c64 sq = pk::mul(x512, x512);
                        const float p512 = 4.0f * (pk::re(sq) + pk::im(sq));
                        p2 = (lane == 0) ? p512 : p2;
                    }
                    float m1 = sqrt_approx(p1), m2 = sqrt_approx(p2);
                    if(EXTRA && p.slope != nullptr)
                    {
                        m1 *= __ldg(p.slope + k1);
                        m2 *= __ldg(p.slope + k2);
                    }
                    mymag[k1] = m1;
                    mymag[k2] = m2;
                }
                if(lane == 0)
                    ctl_nz[wi] = nz ? 1 : 0;
            }
            team::bar_sync(bar_id, W * 32);

            // =================== phase 2: this warp's bin slice through the round's ticks, in order ===================
            // Common case — a full round, every frame has signal, no skip mask: straight-line code for the W ticks (the
            // loads of all ticks issue up front, only the EMA chain is serial), no per-tick gate logic.
            bool round_done = false;
            if(t0 + W <= T && !(EXTRA && p.skip_mask != nullptr))
            {
                bool all_nz = true;
#pragma unroll
                for(int i = 0; i < W; ++i)
                    all_nz &= ctl_nz[i] != 0;
                if(all_nz)
                {
                    last_silent = false;
                    float *odb0 = p.out_db + ((size_t)s * T + t0) * B + b0;
                    float dl[BPL]; // dB of the round's last tick (gate flags)
#pragma unroll
                    for(int i = 0; i < W; ++i)
                    {
                        const int tt = t0 + i;
                        const float2 gt = (EXTRA && p.g_tab != nullptr) ? __ldg(p.g_tab + tt) : make_float2(p.g, p.g2);
                        const float *mg = reinterpret_cast<const float *>(warps_base + (size_t)(tm * W + i) * kWarpBytes + kWarpBufBytes) + b0;
                        float d[BPL];
#pragma unroll
                        for(int j = 0; j < BPL; j += VEC)
                        {
                            float m[4];
                            if constexpr(VEC == 4)
                            {
                                const float4 x = *reinterpret_cast<const float4 *>(mg + j);
                                m[0] = x.x, m[1] = x.y, m[2] = x.z, m[3] = x.w;
                            }
                            else
                            {
                                const float2 x = *reinterpret_cast<const float2 *>(mg + j);
                                m[0] = x.x, m[1] = x.y;
                            }
#pragma unroll
                            for(int u = 0; u < VEC; ++u)
                            {
                                float mm = m[u];
                                if(tsm)
                                {
                                    float old = st[j + u];
                                    if(EXTRA && p.fast_peaks)
                                        old = fmaxf(mm, old);
                                    mm = fmaf(gt.x, old, gt.y * mm);
                                }
                                st[j + u] = mm;
                            }
                        }
#pragma unroll
                        for(int j = 0; j < BPL; j += 2)
                            pk::split(dbfs2(st[j], st[j + 1], p.db_min), d[j], d[j + 1]);
                        if(EXTRA)
                        {
                            float vc = 0.0f;
                            if(p.normalize)
                            {
                                const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + tt] : 0.0f;
                                vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
                            }
                            float peak = -INFINITY;
#pragma unroll
                            for(int j = 0; j < BPL; ++j)
                            {
                                const int k = b0 + j;
                                if(k >= 1)
                                {
                                    if(p.normalize)
                                        d[j] += vc;
                                    if(p.rolloff != nullptr)
                                        d[j] = fmaxf(d[j] - __ldg(p.rolloff + k), p.db_min);
                                    peak = fmaxf(peak, d[j]);
                                }
                            }
                            if(p.out_peak != nullptr)
                            {
                                const float gm = group_max<32>(peak, nullptr);
                                if(lane == 0)
                                    atomic_max_float(p.out_peak + tt, gm);
                            }
                        }
                        float *odb = odb0 + (size_t)i * B;
#pragma unroll
                        for(int j = 0; j < BPL; j += VEC)
                        {
                            if constexpr(VEC == 4)
                                asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(odb + j), "f"(d[j]), "f"(d[j + 1]),
                                             "f"(d[j + 2]), "f"(d[j + 3])
                                             : "memory");
                            else
                                asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(odb + j), "f"(d[j]), "f"(d[j + 1]) : "memory");
                        }
                        if(i == W - 1)
                        {
#pragma unroll
                            for(int j = 0; j < BPL; ++j)
                                dl[j] = d[j];
                        }
                    }
                    if(gate)
                    {
                        bool outs = true;
#pragma unroll
                        for(int j = 0; j < BPL; ++j)
                            outs &= !(dl[j] > p.floor_m10);
                        outs_lane = outs;
                        pos_valid = false;
                    }
                    if(p.out_silent != nullptr && wi == 0 && lane < W)
                        p.out_silent[(size_t)s * T + t0 + lane] = 0;
                    last_from_state = true;
                    round_done = true;
                }
            }
#pragma unroll 1
            for(int i = 0; i < W && !round_done; ++i)
            {
                const int tt = t0 + i;
                if(tt >= T)
                    break;
                const bool nz = ctl_nz[i] != 0;
                const bool skip_all = EXTRA && (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + tt] != 0);
                bool do_proc = !skip_all;
                if(!skip_all)
                {
                    if(nz)
                        last_silent = false;
                    else if(gate)
                    {
                        if(last_silent)
                            do_proc = false;
                        else
                        {
                            if(!pos_valid)
                            {
                                pos = team_all(outs_lane);
                                pos_valid = true;
                            }
                            if(pos)
                            {
                                last_silent = true;
                                do_proc = false;
                            }
                        }
                    }
                }
                const float2 gt = (EXTRA && p.g_tab != nullptr) ? __ldg(p.g_tab + tt) : make_float2(p.g, p.g2); // gravity of this tick
                float *odb = p.out_db + ((size_t)s * T + tt) * B + b0;
                float vc = 0.0f;
                if(EXTRA && p.normalize)
                {
                    const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + tt] : 0.0f;
                    vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
                }
                float d[BPL];
                if(do_proc && !last_silent)
                {
                    const float *mg = reinterpret_cast<const float *>(warps_base + (size_t)(tm * W + i) * kWarpBytes + kWarpBufBytes) + b0;
#pragma unroll
                    for(int j = 0; j < BPL; j += VEC)
                    {
                        float m[4];
                        if constexpr(VEC == 4)
                        {
                            const float4 x = *reinterpret_cast<const float4 *>(mg + j);
                            m[0] = x.x, m[1] = x.y, m[2] = x.z, m[3] = x.w;
                        }
                        else
                        {
                            const float2 x = *reinterpret_cast<const float2 *>(mg + j);
                            m[0] = x.x, m[1] = x.y;
                        }
#pragma unroll
                        for(int u = 0; u < VEC; ++u)
                        {
                            float mm = m[u];
                            if(tsm)
                            {
                                float old = st[j + u];
                                if(EXTRA && p.fast_peaks)
                                    old = fmaxf(mm, old);
                                // one fused rounding, as wf_fast2048.cuh and the reference's AVX2 path (src/source_avx2.cpp:154)
                                mm = fmaf(gt.x, old, gt.y * mm);
                            }
                            st[j + u] = mm;
                        }
                    }
#pragma unroll
                    for(int j = 0; j < BPL; j += 2)
                    {
                        pk::split(dbfs2(st[j], st[j + 1], p.db_min), d[j], d[j + 1]);
                    }
                    if(EXTRA)
                    {
#pragma unroll
                        for(int j = 0; j < BPL; ++j)
                        {
                            const int k = b0 + j;
                            if(k >= 1)
                            {
                                if(p.normalize)
                                    d[j] += vc;
                                if(p.rolloff != nullptr)
                                    d[j] = fmaxf(d[j] - __ldg(p.rolloff + k), p.db_min);
                            }
                        }
                    }
                    last_from_state = true;
                }
                else
                {
                    // tick returned early (hold) or the channel was skipped while the tick went on (stale dB re-converted)
                    const bool from_state = (tt == 0) && hold_lazy;
                    const float *prev_db = (tt > 0) ? (odb - B) : (hold_s + b0);
#pragma unroll
                    for(int j = 0; j < BPL; j += 2)
                    {
                        float o1, o2;
                        if(from_state)
                            pk::split(dbfs2(st[j], st[j + 1], p.db_min), o1, o2);
                        else
                        {
                            o1 = prev_db[j];
                            o2 = prev_db[j + 1];
                        }
                        if(!last_silent)
                        {
                            o1 = dbfs(o1, p.db_min);
                            o2 = dbfs(o2, p.db_min);
                            if(EXTRA)
                            {
                                const int k = b0 + j;
                                if(p.normalize)
                                {
                                    if(k >= 1)
                                        o1 += vc;
                                    o2 += vc;
                                }
                                if(p.rolloff != nullptr)
                                {
                                    if(k >= 1)
                                        o1 = fmaxf(o1 - __ldg(p.rolloff + k), p.db_min);
                                    o2 = fmaxf(o2 - __ldg(p.rolloff + k + 1), p.db_min);
                                }
                            }
                        }
                        d[j] = o1;
                        d[j + 1] = o2;
                    }
                    last_from_state = false;
                }
                bool outs = true;
#pragma unroll
                for(int j = 0; j < BPL; ++j)
                    outs &= !(d[j] > p.floor_m10);
#pragma unroll
                for(int j = 0; j < BPL; j += VEC)
                {
                    if constexpr(VEC == 4)
                        asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(odb + j), "f"(d[j]), "f"(d[j + 1]), "f"(d[j + 2]),
                                     "f"(d[j + 3])
                                     : "memory");
                    else
                        asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(odb + j), "f"(d[j]), "f"(d[j + 1]) : "memory");
                }
                if(gate && !last_silent)
                {
                    outs_lane = outs;
                    pos_valid = false;
                }
                if(p.out_silent != nullptr && wi == 0 && lane == 0)
                    p.out_silent[(size_t)s * T + tt] = last_silent ? 1 : 0;
                if(EXTRA && p.out_peak != nullptr)
                {
                    float peak = -INFINITY;
#pragma unroll
                    for(int j = 0; j < BPL; ++j)
                        if(b0 + j >= 1)
                            peak = fmaxf(peak, d[j]);
                    const float gm = group_max<32>(peak, nullptr);
                    if(lane == 0)
                        atomic_max_float(p.out_peak + tt, gm);
                }
            }
            team::bar_sync(bar_id, W * 32); // every slice has consumed the round's magnitudes
        }

        // ---- state back to the engine; m_decibels mirror (left implicit when it equals dbfs(state)); flags ----
        if(gate && !pos_valid)
            pos = team_all(outs_lane);
        {
            const bool plain = !EXTRA || (!p.normalize && p.rolloff == nullptr);
            const bool lazy = last_from_state && plain && (p.lazy_hold != 0);
            const float *last = p.out_db + ((size_t)s * T + (T - 1)) * B + b0;
#pragma unroll
            for(int j = 0; j < BPL; j += 2)
            {
                *reinterpret_cast<float2 *>(state_s + b0 + j) = make_float2(st[j], st[j + 1]);
                if(p.write_hold && !lazy)
                {
                    float h1, h2;
                    if(last_from_state && plain)
                        pk::split(dbfs2(st[j], st[j + 1], p.db_min), h1, h2);
                    else
                    {
                        h1 = last[j];
                        h2 = last[j + 1];
                    }
                    *reinterpret_cast<float2 *>(hold_s + b0 + j) = make_float2(h1, h2);
                }
            }
            if(wi == 0 && lane == 0)
                p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (pos ? 2u : 0u) | 4u | (lazy ? 8u : 0u));
        }
        __syncwarp();
    }
}

} // namespace wf
