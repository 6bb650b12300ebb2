// wf_par16384.cuh — N = 16384 (BASELINE.json configs[4]), one capture channel, spectrum (+ peak) output:
// a cluster of TWO CTAs per stream that splits the BINS BY PARITY, each CTA running the N=8192 plan without spills.
//
// The CTA-per-tick kernel holds 32 points per thread for this size (radix-2 first stage + two 4096-point sub-FFTs one after the
// other: 128 registers, 346 B of spills, 21 % of the HBM roofline).  One radix-2 decimation-in-frequency stage splits the
// packed 8192-point complex FFT of a frame into
//     rank 0:  e[n] =  z[n] + z[n+4096]                 -> X[2k']   = FFT4096(e)[k']
//     rank 1:  o[n] = (z[n] - z[n+4096]) W_8192^n       -> X[2k'+1] = FFT4096(o)[k']
// and the real-FFT split pairs bin k with 8192-k: even with even (k' <-> 4096-k'), odd with odd (k' <-> 4095-k') — so each CTA
// owns its parity class END TO END (split pass, |X|, slope, EMA state in registers, dBFS, gate flags, stores): no magnitude
// exchange at all.  Both CTAs read the whole frame (the second read is an L2 hit) and therefore see the same "any sample
// non-zero"; the only cluster traffic is the gate's all-bins test, reduced lazily through distributed shared memory when a
// silent tick needs it, and once at the end of the call.  The 4096-point sub-FFT is v3::Fft3<8192>::run_core — 16 points per
// thread, 256 threads, three register passes, every shared-memory access base + immediate (wf_v3.cuh).
// Semantics: src/source_generic.cpp:26-180 as restated in wf_fast2048.cuh / wf_v3.cuh.
#pragma once
#include <cstdint>

#include "wf_v3.cuh"

namespace wf {

namespace par16384 {
constexpr int kN = 16384, kBins = 8192, kSub = 4096; // bins of the frame, complex points per sub-FFT
using F = v3::Fft3<8192>;                            // the sub-FFT's plan (M = 4096 = 16 x 16 x 16)
using G = v3::Geo3<8192>;
constexpr int kTN = G::TN;       // 256 threads
constexpr int kP = G::P;         // 16 points (= bins) per thread
constexpr int kHP = kP / 2;      // bin pairs per thread
constexpr size_t kBufBytes = (((size_t)G::BUF * sizeof(float2)) + 127) / 128 * 128;
constexpr size_t kStageBytes = (size_t)kN * sizeof(float); // the whole frame, TMA-staged one tick ahead (int16: first half)
constexpr size_t smem_bytes() { return kBufBytes + kStageBytes + 16; }
} // namespace par16384

// The body is instantiated once per cluster rank (r = 0: even bins, r = 1: odd bins) so that every bin index, twiddle index and
// output address is a per-thread base + a compile-time offset: with a run-time rank ncu showed 31 % of the 23 062
// warp-instructions per frame in IMAD / MOV / LEA / IADD3 / LOP3 / ISETP (profiles/r02_par16384.txt).
template<bool EXTRA, int r, typename TS>
__device__ __forceinline__ void par16384_body(const KParams &p, const v3::Tw3 &tw, unsigned char *smem_raw, unsigned (*redf)[2])
{
    using namespace par16384;
    constexpr int B = kBins, TN = kTN, P = kP, HP = kHP, MS = kSub;
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);
    using PS = Pcm<TS>;
    const unsigned char *stage = smem_raw + kBufBytes; // frame t: pairs z[n], n < 8192 (float or int16 samples)
    constexpr uint32_t kFrameBytes = PS::frame_bytes(kN);
    uint64_t *mbar = reinterpret_cast<uint64_t *>(smem_raw + kBufBytes + kStageBytes);
    const int tid = threadIdx.x;
    const int s = blockIdx.x >> 1;
    const int T = p.n_frames;
    const bool tsm = p.tsmooth != 0, gate = p.gate != 0;

    // Bins of this thread, in units of k' (index inside the sub-FFT): pair j -> first k1 = tid + j*TN,
    // second k2: rank 0: 4096 - k1 (thread 0, j = 0: k' = 2048, the self-paired bin; 4096 itself does not exist), rank 1: 4095 - k1.
    // Big-transform bin = 2 k' + r.
    auto second_of = [&](int j) -> int {
        if(r == 1)
            return MS - 1 - tid - j * TN;
        return (j == 0 && tid == 0) ? MS / 2 : MS - tid - j * TN;
    };
    float st[P]; // [2j] = bin k1, [2j+1] = bin k2
    {
        const float *sp = p.state + (size_t)s * B;
#pragma unroll
        for(int j = 0; j < HP; ++j)
        {
            st[2 * j] = sp[2 * (tid + j * TN) + r];
            st[2 * j + 1] = sp[2 * second_of(j) + r];
        }
    }
    const unsigned char fl = p.flags[s];
    bool last_silent = (fl & 1u) != 0;
    bool pos = (fl & 2u) != 0, pos_valid = true; // prev_out_silent over ALL bins of the stream, evaluated lazily
    bool part = true;                            // this thread's share of the last producing tick
    unsigned red_par = 0;
    const TS *pcm_s = PS::base(p.pcm) + (size_t)s * p.stream_stride;
    float *hold_s = p.hold_db + (size_t)s * B;

    // cluster-wide AND of the per-thread flags (rare: a silent tick that needs the answer, and once at the end)
    auto ensure_pos = [&]() {
        if(pos_valid)
            return;
        const int mine = __syncthreads_and(part ? 1 : 0);
        if(tid < 2)
            st_cluster_u32(mapa(smem_u32(&redf[red_par][r]), (unsigned)tid), (unsigned)(mine ? 1 : 0));
        cluster_arrive();
        cluster_wait();
        pos = (redf[red_par][0] != 0) && (redf[red_par][1] != 0);
        red_par ^= 1u;
        pos_valid = true;
    };

    // TMA staging (cp.async.bulk + mbarrier) needs 16-byte aligned frames; otherwise the frame is loaded straight from global
    const bool use_tma = (((uintptr_t)pcm_s & 15u) == 0) && ((p.hop & (16 / PS::kBytes - 1)) == 0);
    uint32_t phase = 0;
    if(tid == 0)
    {
        mbar_init(mbar, 1);
        fence_mbarrier_init();
    }
    __syncthreads();
    // distributed shared memory (the lazy gate reduction) may only be addressed once both CTAs of the cluster are running
    cluster_arrive();
    cluster_wait();
    if(use_tma && T > 0 && tid == 0)
    {
        mbar_expect_tx(mbar, kFrameBytes);
        tma_load_1d(const_cast<unsigned char *>(stage), pcm_s, kFrameBytes, mbar);
    }
    const pk::c64 *win = reinterpret_cast<const pk::c64 *>(p.window2) + tid; // pairs (w[2n], w[2n+1]), n = a*TN + tid
    const pk::c64 *tw0 = reinterpret_cast<const pk::c64 *>(tw.tw0) + tid;    // W_8192^(a*TN + tid)
    const pk::c64 *twp = reinterpret_cast<const pk::c64 *>(p.tw_post);       // W_16384^k, k < 8192
    if(!use_tma && T > 0)
        F::prefetch_l2(pcm_s, tid), F::prefetch_l2(pcm_s + kN / 2, tid);

#pragma unroll 1
    for(int t = 0; t < T; ++t)
    {
        const TS *frame = pcm_s + (size_t)t * p.hop;
        // ---- both halves of the frame, window, radix-2 first stage for MY parity ----
        pk::c64 x[P];
        unsigned long long nzbits = 0;
        if(use_tma)
        {
            mbar_wait(mbar, phase);
            phase ^= 1u;
            // (the rank test sits outside the unrolled loops: inside, ptxas if-converts both variants into predicated code)
            if(r == 0)
            {
#pragma unroll
                for(int a = 0; a < P; ++a)
                {
                    pk::c64 za = PS::smem_pair(stage, a * TN + tid), zb = PS::smem_pair(stage, MS + a * TN + tid);
                    nzbits |= za | zb;
                    if(p.window2 != nullptr)
                    {
                        za = pk::mul(za, __ldg(win + a * TN));
                        zb = pk::mul(zb, __ldg(win + MS + a * TN));
                    }
                    x[a] = pk::add(za, zb);
                }
            }
            else
            {
#pragma unroll
                for(int a = 0; a < P; ++a)
                {
                    pk::c64 za = PS::smem_pair(stage, a * TN + tid), zb = PS::smem_pair(stage, MS + a * TN + tid);
                    nzbits |= za | zb;
                    if(p.window2 != nullptr)
                    {
                        za = pk::mul(za, __ldg(win + a * TN));
                        zb = pk::mul(zb, __ldg(win + MS + a * TN));
                    }
                    x[a] = pk::cmul(pk::sub(za, zb), __ldg(tw0 + a * TN));
                }
            }
            __syncthreads(); // every thread has taken its samples: the staging area can receive the next frame
            if(tid == 0 && t + 1 < T)
            {
                fence_proxy_async();
                mbar_expect_tx(mbar, kFrameBytes);
                tma_load_1d(const_cast<unsigned char *>(stage), frame + p.hop, kFrameBytes, mbar);
            }
        }
        else
        {
            const typename PS::Pair *lo = reinterpret_cast<const typename PS::Pair *>(frame) + tid;
            const typename PS::Pair *hi = lo + MS;
#pragma unroll
            for(int a = 0; a < P; ++a)
            {
                pk::c64 za, zb;
                if(p.aligned8)
                {
                    za = pk::from(PS::load2(lo + a * TN));
                    zb = pk::from(PS::load2(hi + a * TN));
                }
                else
                {
                    const TS *f = frame + 2 * (a * TN + tid);
                    za = pk::make(PS::load1(f), PS::load1(f + 1));
                    zb = pk::make(PS::load1(f + 2 * MS), PS::load1(f + 2 * MS + 1));
                }
                nzbits |= za | zb;
                if(p.window2 != nullptr)
                {
                    za = pk::mul(za, __ldg(win + a * TN));
                    zb = pk::mul(zb, __ldg(win + MS + a * TN));
                }
                x[a] = (r == 0) ? pk::add(za, zb) : pk::cmul(pk::sub(za, zb), __ldg(tw0 + a * TN));
            }
            if(t + 1 < T) // next frame -> L2 while this one is transformed
                F::prefetch_l2(frame + p.hop, tid), F::prefetch_l2(frame + p.hop + kN / 2, tid);
        }
        const bool nz = F::template run_core<1, true>(x, buf, tw, tid, (nzbits & 0x7fffffff7fffffffull) != 0ull,
                                                       reinterpret_cast<pk::c64 *>(buf));
        const pk::c64 *X = reinterpret_cast<const pk::c64 *>(buf);

        // ---- gate (src/source_generic.cpp:63-95): both CTAs decide alike (same frame, same flags) ----
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
                else
                {
                    ensure_pos();
                    if(pos)
                    {
                        last_silent = true;
                        do_proc = false;
                    }
                }
            }
        }
        const float2 gt = (EXTRA && p.g_tab != nullptr) ? __ldg(p.g_tab + t) : make_float2(p.g, p.g2);
        float vc = 0.0f;
        if(EXTRA && p.normalize)
        {
            const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + t] : 0.0f;
            vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
        }
        float *odb = p.out_db + ((size_t)s * T + t) * B + r;
        float omax = -INFINITY, peak = -INFINITY;

        if(do_proc && !last_silent)
        {
#pragma unroll
            for(int j = 0; j < HP; ++j)
            {
                const int k1 = tid + j * TN, k2 = second_of(j);
                const pk::c64 a = X[k1];
                const pk::c64 bq = X[(r == 0 && j == 0 && tid == 0) ? 0 : k2];
                const pk::c64 b = pk::conj(bq);
                const pk::c64 sum = pk::add(a, b);
                const pk::c64 o = pk::mul_neg_i(pk::sub(a, b));
                const pk::c64 wo = pk::cmul(o, __ldg(twp + 2 * k1 + r));
                const pk::c64 y1 = pk::add(sum, wo);
                const pk::c64 y2 = pk::sub(sum, wo);
                const pk::c64 s1 = pk::mul(y1, y1), s2 = pk::mul(y2, y2);
                float p1 = pk::re(s1) + pk::im(s1);
                float p2 = pk::re(s2) + pk::im(s2);
                if(j == 0)
                {
                    // rank 0, thread 0: the pair (0, 8192) has no bin 8192; its second slot carries bin 4096 (k' = 2048)
                    const pk::c64 xm = X[MS / 2];
                    const pk::c64 sq = pk::mul(xm, xm);
                    const float pm = 4.0f * (pk::re(sq) + pk::im(sq));
                    p2 = (r == 0 && tid == 0) ? pm : p2;
                }
                pk::c64 m = pk::mul(pk::make(sqrt_approx_ftz(p1), sqrt_approx_ftz(p2)), pk::make(p.coef_half, p.coef_half));
                if(EXTRA && p.slope != nullptr)
                    m = pk::mul(m, pk::make(__ldg(p.slope + 2 * k1 + r), __ldg(p.slope + 2 * k2 + r)));
                if(tsm)
                {
                    pk::c64 old = pk::make(st[2 * j], st[2 * j + 1]);
                    if(EXTRA && p.fast_peaks)
                        old = pk::make(fmaxf(pk::re(m), st[2 * j]), fmaxf(pk::im(m), st[2 * j + 1]));
                    m = pk::fma(pk::make(gt.x, gt.x), old, pk::mul(pk::make(gt.y, gt.y), m)); // as wf_v3.cuh / wf_fast2048.cuh
                }
                pk::split(m, st[2 * j], st[2 * j + 1]);
                float d1, d2;
                pk::split(dbfs2(st[2 * j], st[2 * j + 1], p.db_min), d1, d2);
                if(EXTRA)
                {
                    if(p.normalize)
                    {
                        if(2 * k1 + r >= 1)
                            d1 += vc;
                        d2 += vc;
                    }
                    if(p.rolloff != nullptr)
                    {
                        if(2 * k1 + r >= 1)
                            d1 = fmaxf(d1 - __ldg(p.rolloff + 2 * k1 + r), p.db_min);
                        d2 = fmaxf(d2 - __ldg(p.rolloff + 2 * k2 + r), p.db_min);
                    }
                    if(2 * k1 + r >= 1)
                        peak = fmaxf(peak, d1);
                    peak = fmaxf(peak, d2);
                }
                omax = fmaxf(omax, fmaxf(d1, d2));
                stg_stream(odb + 2 * k1, d1);
                stg_stream(odb + 2 * k2, d2);
            }
        }
        else
        {
            // tick returned early (hold) or the channel was skipped while the tick went on (stale dB re-converted)
            const float *prev_db = (t > 0) ? (odb - B) : (hold_s + r);
#pragma unroll 1
            for(int j = 0; j < HP; ++j)
            {
#pragma unroll
                for(int h = 0; h < 2; ++h)
                {
                    const int k = 2 * (h == 0 ? tid + j * TN : second_of(j));
                    float o = prev_db[k];
                    if(!last_silent)
                    {
                        o = dbfs(o, p.db_min);
                        if(EXTRA && k + r >= 1)
                        {
                            if(p.normalize)
                                o += vc;
                            if(p.rolloff != nullptr)
                                o = fmaxf(o - __ldg(p.rolloff + k + r), p.db_min);
                        }
                    }
                    omax = fmaxf(omax, o);
                    if(k + r >= 1)
                        peak = fmaxf(peak, o);
                    odb[k] = o;
                }
            }
        }
        if(gate && !last_silent)
        {
            part = !(omax > p.floor_m10);
            pos_valid = false;
        }
        if(p.out_silent != nullptr && r == 0 && tid == 0)
            p.out_silent[(size_t)s * T + t] = last_silent ? 1 : 0;
        if(EXTRA && p.out_peak != nullptr)
        {
            __shared__ float red_scratch[TN / 32];
            const float gm = group_max<TN>(peak, red_scratch);
            if(tid == 0)
                atomic_max_float(p.out_peak + t, gm);
        }
        // (the next frame's FFT starts with a block barrier before it overwrites the buffer)
    }

    // ---- state back to the engine; m_decibels mirror; flags ----
    ensure_pos();
    {
        float *sp = p.state + (size_t)s * B;
#pragma unroll
        for(int j = 0; j < HP; ++j)
        {
            sp[2 * (tid + j * TN) + r] = st[2 * j];
            sp[2 * second_of(j) + r] = st[2 * j + 1];
        }
        if(p.write_hold && T > 0)
        {
            const float *last = p.out_db + ((size_t)s * T + (T - 1)) * B + r;
#pragma unroll
            for(int j = 0; j < HP; ++j)
            {
                const int k1 = 2 * (tid + j * TN), k2 = 2 * second_of(j);
                hold_s[k1 + r] = last[k1];
                hold_s[k2 + r] = last[k2];
            }
        }
        if(r == 0 && tid == 0)
            p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (pos ? 2u : 0u) | 4u);
    }
    cluster_arrive(); // no CTA may exit while its peer can still address its shared memory
    cluster_wait();
}

template<bool EXTRA, typename TS>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(par16384::kTN, 2)
    stft16384_parity_kernel(const __grid_constant__ KParams p, const __grid_constant__ v3::Tw3 tw)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ unsigned redf[2][2]; // [parity of the exchange][rank]: this rank's "all my outputs <= floor-10 dB"
    if(cluster_ctarank() == 0)
        par16384_body<EXTRA, 0, TS>(p, tw, smem_raw, redf);
    else
        par16384_body<EXTRA, 1, TS>(p, tw, smem_raw, redf);
}

} // namespace wf
