// wf_warp2.cuh — the warp-per-stream kernel of wf_fast2048.cuh generalised to fft sizes N = 2*L*P with L, P <= 32:
// the plugin's NON-POWER-OF-TWO sizes (SURVEY §8(f) rank 1): the automatic size sr/fps & -16 (800 at 48 kHz / 60 fps,
// 720, 960, 1600, 1456 ...) and the slider's 64-sample steps up to 2048 (src/source.cpp:349,562-565,1161-1167).
//
// One WARP owns one stream and walks its frames; per frame (M = N/2 = L*P packed complex points, n = n1 + L*n2):
//   * the N*4-byte PCM frame is staged HBM -> shared memory by a TMA bulk copy (cp.async.bulk + mbarrier), one frame ahead;
//   * pass A: lane n1 < L holds the P points n2 = 0..P-1 and runs a radix-P REGISTER DFT (pk::dft_mixed: radix 2 / 3 / 5 /
//     7 / 11 / 13 butterflies with compile-time twiddles); inter-pass twiddle W_M^(n1 k2) from a shared table; ONE padded
//     shared-memory transpose;
//   * pass B: lane k2 < P holds the L points n1 = 0..L-1 and runs a radix-L register DFT -> X[k2 + P k1];
//   * the real-FFT split pass handles bins k and M-k together (partner value by warp shuffle from lane (P-k2) % P), |X| via
//     MUFU.SQRT, slope, EMA (state in shared memory across the stream's frames), dBFS via MUFU.LG2, gate / hold / skip /
//     volume / roll-off exactly as wf_fast2048.cuh; stores are runs of P consecutive floats.
// The first-generation any-N kernel (wf_anyn.cuh: run-time O(M * sum r) DFT passes, 4-5 % of the HBM roofline) remains the
// fallback for sizes without such a factorisation (N > 2048 or a prime factor > 13 in the wrong place) and for display outputs.
#pragma once
#include <type_traits>

#include "wf_kernels.cuh"

namespace wf {

namespace warp2 {

constexpr int imax(int a, int b) { return a > b ? a : b; }

// compile-time loop: f(std::integral_constant<int, I>) for I = I0 .. I1-1 (register indices must be constants)
template<int I0, int I1, class F>
__device__ __forceinline__ void static_for(F &&f)
{
    if constexpr(I0 < I1)
    {
        f(std::integral_constant<int, I0>{});
        static_for<I0 + 1, I1>(f);
    }
}

template<int L, int P>
struct Geo {
    static constexpr int M = L * P;
    static constexpr int N = 2 * M;
    static constexpr int R = imax(L, P);                 // complex registers per lane
    static constexpr int PP = P + ((P % 2 == 0) ? 1 : 0); // padded row of the transpose buffer (odd -> conflict-free 64-bit)
    static constexpr int Q = (L + 1) / 2;                // bin pairs per lane
    static constexpr int kBufElems = imax(M, L * PP);    // float2 elements: TMA landing zone and transpose area
    static constexpr int kBufBytes = ((kBufElems * 8 + 127) / 128) * 128;
    static constexpr int kStateBytes = ((Q * 32 * 8 + 127) / 128) * 128; // [q][lane] -> (first bin, second bin)
    static constexpr int kWarpBytes = kBufBytes + kStateBytes + 128;      // + mbarrier (keeps 128-byte alignment)
    static constexpr int kTableElems = M /*window*/ + M /*twA*/ + Q * 32 /*twP*/;
    static constexpr int kTableBytes = ((kTableElems * 8 + 127) / 128) * 128;
    static constexpr int kWarps = 16;
    static constexpr int smem_bytes(int warps) { return kTableBytes + warps * kWarpBytes; }
};

} // namespace warp2

// DISP: the render-time stages (interpolation to curve points / bars, Gaussian, pixels, running minimum; display_stage<32> of
// wf_kernels.cuh, the one the CTA-per-tick kernels use) run on the warp right after the tick's dB row, which is then kept
// in a per-warp shared-memory row (it doubles as the "previous row" of the hold paths; out_db may be null).  The extra
// per-warp area (p.disp_bytes: dB row, display scratch, arg-min scratch) follows the regular per-warp areas.
template<int L, int P, bool EXTRA, bool DISP, typename TS>
__global__ void __launch_bounds__(warp2::Geo<L, P>::kWarps * 32, 1) stft_warp2_kernel(const __grid_constant__ KParams p)
{
    using G = warp2::Geo<L, P>;
    using PS = Pcm<TS>;
    constexpr int M = G::M, N = G::N, R = G::R, PP = G::PP, Q = G::Q, B = M;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2 *s_win = reinterpret_cast<float2 *>(smem_raw); // window pairs (x[2n], x[2n+1]) * (2/sum(w))/2
    float2 *s_twA = s_win + M;                            // [k2][n1] = W_M^(k2*n1)
    float2 *s_twP = s_twA + M;                            // [q][lane] = W_N^(lane + P q)
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int warps_per_cta = blockDim.x >> 5;
    unsigned char *wbase = smem_raw + G::kTableBytes + warp * G::kWarpBytes;
    float2 *buf = reinterpret_cast<float2 *>(wbase);
    float2 *sst = reinterpret_cast<float2 *>(wbase + G::kBufBytes) + lane;
    uint64_t *mbar = reinterpret_cast<uint64_t *>(wbase + G::kBufBytes + G::kStateBytes);
    // DISP: [CTA: interpolation weights | indices | Gaussian | band widths | band offsets] (p.disp_tab_bytes, copied once
    // below: a persistent CTA reads them n_points times per warp and tick) then per warp [dB row | bar samples | points x 2 |
    // arg-min scratch] (p.disp_bytes; the last two only for the Gaussian / pixel / minimum outputs) — wf_engine.cu sizes both
    float *dbs = nullptr, *disp_tmp = nullptr, *disp_pts = nullptr, *disp_red = nullptr;
    DispTab dtab{};
    if constexpr(DISP)
    {
        unsigned char *db0 = smem_raw + G::kTableBytes + (size_t)warps_per_cta * G::kWarpBytes;
        dtab = stage_display_tables(p, reinterpret_cast<float *>(db0), threadIdx.x, blockDim.x);
        const bool need_pts = p.filter || (p.out_pixels != nullptr) || (p.out_min != nullptr);
        dbs = reinterpret_cast<float *>(db0 + p.disp_tab_bytes + (size_t)warp * p.disp_bytes);
        disp_tmp = dbs + B;
        disp_pts = disp_tmp + p.n_sample;
        disp_red = disp_pts + (need_pts ? 2 * p.n_points : 0);
    }

    for(int i = threadIdx.x; i < M; i += blockDim.x)
    {
        const float2 w = (p.window2 != nullptr) ? __ldg(p.window2 + i) : make_float2(1.0f, 1.0f);
        s_win[i] = make_float2(w.x * p.coef_half, w.y * p.coef_half);
        s_twA[i] = __ldg(p.tw + (((i / L) * (i % L)) % M)); // i = k2*L + n1
    }
    for(int i = threadIdx.x; i < Q * 32; i += blockDim.x)
    {
        const int k = (i & 31) + P * (i >> 5);
        s_twP[i] = ((i & 31) < P && k < M) ? __ldg(p.tw_post + k) : make_float2(1.0f, 0.0f);
    }
    int *seg_done = reinterpret_cast<int *>(mbar + 1); // split mode: this warp's head segment is finished
    if(lane == 0)
    {
        mbar_init(mbar, 1);
        *seg_done = 0;
        fence_mbarrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    const int S = p.n_streams, T = p.n_frames;
    const int GR = gridDim.x;
    const int n_local = (S > (int)blockIdx.x) ? (S - (int)blockIdx.x + GR - 1) / GR : 0;
    uint32_t phase = 0;
    const bool tsm = p.tsmooth != 0, gate = p.gate != 0;

    const bool act_a = lane < L;              // pass A: lane = n1
    const bool act_b = lane < P;              // pass B and epilogue: lane = k2
    const int la = act_a ? lane : 0;          // keeps the idle lanes' addresses inside the buffers
    const int lb = act_b ? lane : 0;
    const int jp = (P - lb) % P;              // partner lane of the split pass
    // second bin of pair q: lane != 0: (P - lane) + P (L-1-q); lane 0: P (L - q) (q >= 1); q == 0 on lane 0: M/2 if L is even
    const int kb2 = (lb == 0) ? 0 : (P - lb);

    // ---- work list of this warp: whole streams dealt round-robin, or (split mode, see wf_fast2048.cuh) the SM's n_local * T
    // frames cut into equal runs [tail of stream a][whole streams][head of stream b]; a stream changes warps through global
    // memory (state, flags, mirror) behind a shared-memory flag, exactly as it would between two calls ----
    const int rounds_whole = (n_local + warps_per_cta - 1) / warps_per_cta;
    const bool split = (p.split != 0) && (n_local >= warps_per_cta) && (T > 1) &&
                       (2 * (rounds_whole * warps_per_cta - n_local) * T > 3 * warps_per_cta);
    int u0 = 0, u1 = 0;
    if(split)
    {
        const int U = n_local * T, per = (U + warps_per_cta - 1) / warps_per_cta;
        u0 = min(warp * per, U);
        u1 = min(u0 + per, U);
    }
    const int full0 = (u0 + T - 1) / T, full1 = u1 / T;
    const int has_head = (split && (u1 % T) != 0) ? 1 : 0, has_tail = (split && (u0 % T) != 0) ? 1 : 0;
    const int nseg = split ? (has_head + max(full1 - full0, 0) + has_tail)
                           : ((n_local > warp) ? (n_local - warp + warps_per_cta - 1) / warps_per_cta : 0);
    auto segment = [&](int j, int &li, int &t0, int &t1) {
        if(!split)
        {
            li = warp + j * warps_per_cta;
            t0 = 0;
            t1 = T;
            return;
        }
        if(has_head && j == 0)
        {
            li = full1;
            t0 = 0;
            t1 = u1 % T;
            return;
        }
        j -= has_head;
        if(j < full1 - full0)
        {
            li = full0 + j;
            t0 = 0;
            t1 = T;
            return;
        }
        li = u0 / T;
        t0 = u0 % T;
        t1 = T;
    };

    if(nseg > 0 && lane == 0)
    {
        int li, t0, t1;
        segment(0, li, t0, t1);
        mbar_expect_tx(mbar, PS::frame_bytes(N));
        tma_load_1d(buf, PS::base(p.pcm) + (size_t)(blockIdx.x + li * GR) * p.stream_stride + (size_t)t0 * p.hop, PS::frame_bytes(N),
                    mbar);
    }

    for(int j = 0; j < nseg; ++j)
    {
        int li, t0, t1;
        segment(j, li, t0, t1);
        const int s = (int)blockIdx.x + li * GR;
        int s_next = -1, t0_next = 0;
        if(j + 1 < nseg)
        {
            int li2, t12;
            segment(j + 1, li2, t0_next, t12);
            s_next = (int)blockIdx.x + li2 * GR;
        }
        if(t0 > 0)
        {
            // continuation of a stream whose first ticks the previous warp ran as its head segment
            int *prev_done = reinterpret_cast<int *>(wbase - G::kWarpBytes + G::kBufBytes + G::kStateBytes + 8);
            if(lane == 0)
                while(atomicAdd(prev_done, 0) == 0)
                    ;
            __syncwarp();
            __threadfence_block();
        }
        float *state_s = p.state + (size_t)s * B;
        // second-bin index of this lane for pair q (negative = no such bin)
        auto k2_of = [&](int q) -> int {
            if(lb != 0) // the middle pair of an odd L shows up on both lanes k2 and P-k2: each keeps only its FIRST bin
                return ((L % 2 == 1) && (q == (L - 1) / 2)) ? -1 : kb2 + P * (L - 1 - q);
            if(q == 0)
                return (L % 2 == 0) ? (M / 2) : -1;
            return P * (L - q);
        };
        // ---- per-stream state: global (natural bin order) -> shared ([pair][lane]) ----
        if(act_b)
        {
#pragma unroll
            for(int q = 0; q < Q; ++q)
            {
                const int k1 = lane + P * q;
                const int k2 = k2_of(q);
                sst[q * 32] = make_float2(state_s[k1], (k2 >= 0) ? state_s[k2] : 0.0f);
            }
        }
        const unsigned char fl = p.flags[s];
        bool last_silent = (fl & 1u) != 0;
        bool prev_out_silent = (fl & 2u) != 0;
        const TS *pcm_s = PS::base(p.pcm) + (size_t)s * p.stream_stride;
        float *hold_s = p.hold_db + (size_t)s * B;

#pragma unroll 1
        for(int t = t0; t < t1; ++t)
        {
            mbar_wait(mbar, phase);
            phase ^= 1u;
            pk::c64 v[R];
            unsigned long long nzbits = 0;
            const pk::c64 *buf64 = reinterpret_cast<const pk::c64 *>(buf);
            const pk::c64 *win64 = reinterpret_cast<const pk::c64 *>(s_win);
#pragma unroll
            for(int pi = 0; pi < P; ++pi)
            {
                v[pi] = PS::smem_pair(buf, la + L * pi);
                nzbits |= act_a ? v[pi] : 0ull;
            }
#pragma unroll
            for(int pi = 0; pi < P; ++pi)
                v[pi] = pk::mul(v[pi], win64[la + L * pi]);
            const bool nz = __any_sync(0xffffffffu, (nzbits & 0x7fffffff7fffffffull) != 0ull);

            // ---- pass A: radix-P register DFT over n2, twiddle W_M^(n1 k2), transpose ----
            pk::dft_mixed<P, R>(v);
            __syncwarp(); // every lane has read the frame before the buffer becomes the transpose area
            if(act_a)
            {
                warp2::static_for<0, P>([&](auto kc) {
                    constexpr int k2 = decltype(kc)::value;
                    pk::c64 a = v[pk::perm_mixed(P, k2)];
                    if constexpr(k2 > 0)
                        a = pk::cmul(a, reinterpret_cast<const pk::c64 *>(s_twA)[k2 * L + lane]);
                    reinterpret_cast<pk::c64 *>(buf)[lane * PP + k2] = a;
                });
            }
            __syncwarp();
#pragma unroll
            for(int n1 = 0; n1 < L; ++n1)
                v[n1] = buf64[n1 * PP + lb];
            __syncwarp(); // all generic-proxy accesses to buf are done: it can take the next frame
            if(t + 1 == t1 && s_next >= 0 && t0_next == 0)
                prefetch_l2_line(p.state + (size_t)s_next * B + (lane * 32) % B);
            if(lane == 0)
            {
                const TS *next = nullptr;
                if(t + 1 < t1)
                    next = pcm_s + (size_t)(t + 1) * p.hop;
                else if(s_next >= 0)
                    next = PS::base(p.pcm) + (size_t)s_next * p.stream_stride + (size_t)t0_next * p.hop;
                if(next != nullptr)
                {
                    fence_proxy_async();
                    mbar_expect_tx(mbar, PS::frame_bytes(N));
                    tma_load_1d(buf, next, PS::frame_bytes(N), mbar);
                }
            }
            // ---- pass B: radix-L register DFT over n1: X[k2 + P k1] = v[perm(L, k1)] on lane k2 ----
            pk::dft_mixed<L, R>(v);

            // ---- gate (src/source_generic.cpp:63-95), single capture channel ----
            const bool skip_all = EXTRA && (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + t] != 0);
            bool do_proc = !skip_all;
            if(!skip_all)
            {
                if(nz)
                    last_silent = false;
                else if(gate)
                {
                    if(last_silent)
                        do_proc = false;
                    else if(prev_out_silent)
                    {
                        last_silent = true;
                        do_proc = false;
                    }
                }
            }
            const bool wr_db = !DISP || (p.out_db != nullptr);
            float *odb = wr_db ? p.out_db + ((size_t)s * T + t) * B : nullptr;
            float vc = 0.0f;
            if(EXTRA && p.normalize)
            {
                const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + t] : 0.0f;
                vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
            }
            bool outs = true;
            float peak = -INFINITY;
            const float2 gt = (EXTRA && p.g_tab != nullptr) ? __ldg(p.g_tab + t) : make_float2(p.g, p.g2); // gravity of this tick

            if(do_proc && !last_silent)
            {
                warp2::static_for<0, Q>([&](auto qc) {
                    constexpr int q = decltype(qc)::value;
                    const int k1 = lb + P * q;
                    const int k2 = k2_of(q);
                    const pk::c64 a = v[pk::perm_mixed(L, q)];
                    unsigned long long bp = __shfl_sync(0xffffffffu, v[pk::perm_mixed(L, L - 1 - q)], jp);
                    if(lb == 0)
                        bp = v[pk::perm_mixed(L, (L - q) % L)];
                    const pk::c64 b = pk::conj(bp);
                    const pk::c64 sum = pk::add(a, b);
                    const pk::c64 o = pk::mul_neg_i(pk::sub(a, b));
                    const pk::c64 wo = pk::cmul(o, reinterpret_cast<const pk::c64 *>(s_twP)[q * 32 + lane]);
                    const pk::c64 y1 = pk::add(sum, wo);
                    const pk::c64 y2 = pk::sub(sum, wo);
                    const pk::c64 s1 = pk::mul(y1, y1), s2 = pk::mul(y2, y2);
                    float p1 = pk::re(s1) + pk::im(s1);
                    float p2 = pk::re(s2) + pk::im(s2);
                    if constexpr(q == 0 && (L % 2 == 0))
                    {
                        // lane 0: the pair (0, M) has no bin M; its second slot carries bin M/2 = conj(X[M/2]) doubled
                        const pk::c64 xh = v[pk::perm_mixed(L, L / 2)];
                        const pk::c64 sq = pk::mul(xh, xh);
                        const float ph = 4.0f * (pk::re(sq) + pk::im(sq));
                        p2 = (lb == 0) ? ph : p2;
                    }
                    pk::c64 m = pk::make(sqrt_approx_ftz(p1), sqrt_approx_ftz(p2));
                    const int k2c = (k2 >= 0) ? k2 : 0;
                    if(EXTRA && p.slope != nullptr)
                        m = pk::mul(m, pk::make(__ldg(p.slope + k1), __ldg(p.slope + k2c)));
                    pk::c64 *sst64 = reinterpret_cast<pk::c64 *>(sst);
                    if(tsm)
                    {
                        pk::c64 old = sst64[q * 32];
                        if(EXTRA && p.fast_peaks)
                            old = pk::make(fmaxf(pk::re(m), pk::re(old)), fmaxf(pk::im(m), pk::im(old)));
                        m = pk::fma(pk::make(gt.x, gt.x), old, pk::mul(pk::make(gt.y, gt.y), m));
                    }
                    sst64[q * 32] = m;
                    float d1, d2;
                    pk::split(dbfs2(pk::re(m), pk::im(m), p.db_min), d1, d2);
                    if(EXTRA)
                    {
                        if(p.normalize)
                        {
                            if(k1 >= 1)
                                d1 += vc;
                            d2 += vc;
                        }
                        if(p.rolloff != nullptr)
                        {
                            if(k1 >= 1)
                                d1 = fmaxf(d1 - __ldg(p.rolloff + k1), p.db_min);
                            d2 = fmaxf(d2 - __ldg(p.rolloff + k2c), p.db_min);
                        }
                    }
                    // idle lanes (lane >= P) run the same arithmetic on don't-care values; only the stores are predicated and
                    // the lane's flags are discarded after the loop (no branches inside the unrolled epilogue)
                    const bool st2 = act_b && (k2 >= 0);
                    if(k1 >= 1)
                        peak = fmaxf(peak, d1);
                    outs &= !(d1 > p.floor_m10);
                    if(act_b && wr_db)
                        stg_stream(odb + k1, d1);
                    peak = (k2 >= 0) ? fmaxf(peak, d2) : peak;
                    outs &= (k2 < 0) | !(d2 > p.floor_m10);
                    if(st2 && wr_db)
                        stg_stream(odb + k2c, d2);
                    if constexpr(DISP)
                    {
                        if(act_b)
                            dbs[k1] = d1;
                        if(st2)
                            dbs[k2c] = d2;
                    }
                });
                outs |= !act_b;
                peak = act_b ? peak : -INFINITY;
            }
            else
            {
                // tick returned early (hold) or the channel was skipped while the tick went on (stale dB re-converted)
                // the previous tick's row: the output row, or (DISP) the row kept in shared memory; at the first tick of a
                // segment the mirror, which the previous call — or the warp that ran the stream's first ticks — left behind
                const float *prev_db = (t > t0) ? (DISP ? dbs : (odb - B)) : hold_s;
#pragma unroll 1
                for(int k = lane; k < B; k += 32)
                {
                    float o = prev_db[k];
                    if(!last_silent)
                    {
                        o = dbfs(o, p.db_min);
                        if(EXTRA && k >= 1)
                        {
                            if(p.normalize)
                                o += vc;
                            if(p.rolloff != nullptr)
                                o = fmaxf(o - __ldg(p.rolloff + k), p.db_min);
                        }
                    }
                    outs &= !(o > p.floor_m10);
                    if(k >= 1)
                        peak = fmaxf(peak, o);
                    if(wr_db)
                        odb[k] = o;
                    if constexpr(DISP)
                        dbs[k] = o;
                }
            }
            if constexpr(DISP)
            {
                __syncwarp();
                display_stage_tab<32, false>(p, dtab, dbs, disp_pts, disp_tmp, B, 1, (size_t)s * T + t, lane, true, disp_red);
                __syncwarp();
            }
            if(gate && !last_silent)
                prev_out_silent = __all_sync(0xffffffffu, outs);
            if(p.out_silent != nullptr && lane == 0)
                p.out_silent[(size_t)s * T + t] = last_silent ? 1 : 0;
            if(EXTRA && p.out_peak != nullptr)
            {
                const float gm = group_max<32>(peak, nullptr);
                if(lane == 0)
                    atomic_max_float(p.out_peak + t, gm);
            }
        }

        // ---- state back to the engine; m_decibels mirror for the next call's gate / hold paths ----
        __syncwarp();
        if(act_b)
        {
#pragma unroll
            for(int q = 0; q < Q; ++q)
            {
                const int k1 = lane + P * q;
                const int k2 = k2_of(q);
                const float2 stv = sst[q * 32];
                state_s[k1] = stv.x;
                if(k2 >= 0)
                    state_s[k2] = stv.y;
            }
        }
        if(p.write_hold && T > 0)
        {
            const float *last = DISP ? dbs : p.out_db + ((size_t)s * T + (t1 - 1)) * B;
            __syncwarp();
            for(int k = lane; k < B; k += 32)
                hold_s[k] = last[k];
        }
        if(lane == 0)
            p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (prev_out_silent ? 2u : 0u) | 4u);
        if(t1 < T)
        {
            // head segment: hand the stream to the next warp (state, flags, mirror and output rows are written)
            __threadfence_block();
            __syncwarp();
            if(lane == 0)
                atomicExch(seg_done, 1);
        }
        __syncwarp();
    }
}

} // namespace wf
