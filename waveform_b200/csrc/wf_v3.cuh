// wf_v3.cuh — the fused spectrum pipeline for fft sizes 1024 ... 16384 (powers of two): one CTA per tick, a cluster of R CTAs
// (R = 1, 2, 4, 8) per stream, and a three-pass register FFT whose every shared-memory access is base + immediate.
//
// ncu on the first-generation kernels (profiles/r01i_generic8192.txt) showed 16 750 warp-instructions per N=8192 frame,
// only ~5 000 of them floating point: Stockham index arithmetic (LEA/IMAD/ISETP), run-time flag tests and twiddle loads
// through computed global addresses dominated, with 7 block barriers per frame.  This kernel restructures the same
// mathematics so that the integer work disappears:
//
//   * the N/2-point complex FFT is a 3-D decimation: M = A*B*C, input n = a*BC + b*C + c, output k = ka + A*kb + AB*kc;
//     each pass is a register DFT along one axis (radix A, B, C = 16/32, 16, 8/16) and between passes the data crosses
//     shared memory in layouts chosen so that thread->address is (one base register) + (compile-time offset) and every
//     64-bit access is bank-conflict free:   L1[ka][b][c] (stride BC+pad)  ->  L2[kb][ka][c] (strides A*(C+1), C+1)  ->  X[k];
//   * inter-pass twiddles come from two small tables laid out [index][thread] (tw1[ka][t] = W_M^(t*ka), tw2[kb][c] =
//     W_BC^(c*kb)), i.e. again base + immediate, coalesced, L1-resident;
//   * the real-FFT split pass handles bins k and M-k together (one twiddle multiply for two bins, as wf_fast2048.cuh);
//   * rarely used features (slope, roll-off, volume, fast peaks, skip mask, peak output) are compiled out by template.
//
// Work decomposition is that of wf_wide.cuh (which this kernel supersedes for these sizes): per round of R ticks, CTA r
// transforms tick t0+r, the linear magnitudes are exchanged through distributed shared memory so that CTA q owns bins
// [q*B/R, (q+1)*B/R) of all R ticks, and walks them through the ticks in order with the EMA state in registers.  R = 1
// needs no exchange: the EMA runs on the registers the split pass produced.  HBM traffic is the algorithmic minimum.
// Reference semantics: src/source_generic.cpp:26-180 (see wf_fused.cuh for the line-by-line citations).
#pragma once
#include "wf_kernels.cuh"
#include "wf_v3.hpp"

namespace wf {
namespace v3 {

template<int N> struct Plan3;
template<> struct Plan3<1024> { static constexpr int A = 8, B = 8, C = 8; };
template<> struct Plan3<2048> { static constexpr int A = 16, B = 8, C = 8; };
template<> struct Plan3<4096> { static constexpr int A = 16, B = 16, C = 8; };
template<> struct Plan3<8192> { static constexpr int A = 16, B = 16, C = 16; };
// 16384: a radix-2 first stage in registers, then TWO 4096-point sub-FFTs with the 8192 plan (32 points per thread as one
// radix-32 pass spilled at 128 registers: the window and 31 twiddles are live next to the 32 points).  A = 32 only describes
// the load pattern (32 points per thread, stride TN = 256).
template<> struct Plan3<16384> { static constexpr int A = 32, B = 16, C = 16; };

template<int N>
struct Geo3 {
    static constexpr int M = N / 2;
    static constexpr int A = Plan3<N>::A, B = Plan3<N>::B, C = Plan3<N>::C;
    static_assert(A * B * C == M, "plan does not factor N/2");
    static constexpr int TN = B * C;  // threads per CTA = lines of pass 1
    static constexpr int P = A;       // complex points (= bins) per thread
    static constexpr int LB = A / B;  // lines per thread in pass 2 (A*C lines of B points)
    static constexpr int LC = A / C;  // lines per thread in pass 3 (A*B lines of C points)
    static_assert(LB >= 1 && LC >= 1 && TN % A == 0, "plan shape");
    static constexpr int S1 = B * C + ((C < 16) ? C : 0); // L1 stride per ka (padding keeps half-warps conflict free)
    static constexpr int SA = C + 1;                      // L2 stride per ka
    static constexpr int SB = A * SA;                     // L2 stride per kb
    static constexpr int L1_ELEMS = A * S1;
    static constexpr int L2_ELEMS = B * SB;
    static constexpr bool SPLIT2 = (N == 16384);
    static constexpr int WORK = (L1_ELEMS > L2_ELEMS ? L1_ELEMS : L2_ELEMS);
    // one buffer serves L1, L2, X and the inbox; the split plan keeps X[M] apart from the sub-FFTs' work buffer
    static constexpr int BUF = SPLIT2 ? (M + (B * (A / 2) * (C + 1) > (A / 2) * B * C ? B * (A / 2) * (C + 1) : (A / 2) * B * C)) : WORK;
#ifndef WF_V3_TPSM
#define WF_V3_TPSM 512
#endif
    static constexpr int TPSM = (P <= 8) ? 1024 : WF_V3_TPSM; // resident threads per SM the register cap allows (64 / 128 registers)
    static constexpr int MINB = (TPSM / TN) > 0 ? (TPSM / TN) : 1;
};

// Cluster sizes > 1 with N <= 8192 keep the magnitude inbox in its own double-buffered array: one cluster barrier per round
// instead of two (at 16384 that memory would halve the CTAs per SM, so the inbox aliases the FFT buffer there).
template<int N>
constexpr bool dbuf_inbox() { return N <= 8192; }

// dynamic shared memory of one CTA (cc = capture channels, R = cluster size)
template<int N>
constexpr size_t smem_bytes(int dch, int n_points, bool display, int cc, int R)
{
    size_t b = (size_t)Geo3<N>::BUF * sizeof(float2);
    if(R > 1 && dbuf_inbox<N>())
        b += (size_t)2 * cc * (N / 2) * sizeof(float);
    if(display)
        b += (size_t)dch * (N / 2) * sizeof(float) + (size_t)4 * n_points * sizeof(float);
    return b;
}

// ---- the 3-pass FFT: v[a] = x[a*BC + tid] (windowed) on entry; on exit X[k] sits in buf[k] (natural order) -------
template<int N>
struct Fft3 {
    using G = Geo3<N>;
    static constexpr int M = G::M, A = G::A, B = G::B, C = G::C, TN = G::TN, P = G::P;

    template<typename TS>
    static __device__ __forceinline__ void load_raw(float2 (&v)[P], const TS *frame, int aligned8, int tid)
    {
        using PS = Pcm<TS>;
        if(aligned8)
        {
            const typename PS::Pair *f2 = reinterpret_cast<const typename PS::Pair *>(frame) + tid;
#pragma unroll
            for(int a = 0; a < A; ++a)
                v[a] = PS::load2(f2 + a * TN);
        }
        else
        {
            const TS *f1 = frame + 2 * tid;
#pragma unroll
            for(int a = 0; a < A; ++a)
                v[a] = make_float2(PS::load1(f1 + 2 * a * TN), PS::load1(f1 + 2 * a * TN + 1));
        }
    }
    // pull a frame's cache lines into L2 (when there is no register room for a register prefetch)
    template<typename TS>
    static __device__ __forceinline__ void prefetch_l2(const TS *frame, int tid)
    {
        for(int l = tid; l < N * Pcm<TS>::kBytes / 128; l += TN)
            prefetch_l2_line(frame + l * (128 / Pcm<TS>::kBytes));
    }
    // non-zero test (src/source_generic.cpp:63-76) + window multiply (:97-103); returns "any sample non-zero" (this thread).
    // Split plan: the radix-2 first stage is fused in, pair by pair, so that window and twiddle values die immediately:
    // x[a] = lo + hi (even bins' sub-FFT input), x[a + P/2] = (lo - hi) W_M^(a*TN + tid) (odd bins').
    static __device__ __forceinline__ bool finish_load(pk::c64 (&x)[P], const float2 (&v)[P], const float2 *window2, int tid,
                                                       const Tw3 &tw)
    {
        unsigned long long nzbits = 0;
        if constexpr(!G::SPLIT2)
        {
#pragma unroll
            for(int a = 0; a < A; ++a)
            {
                x[a] = pk::from(v[a]);
                nzbits |= x[a];
            }
            if(window2 != nullptr)
            {
                const pk::c64 *w = reinterpret_cast<const pk::c64 *>(window2) + tid;
#pragma unroll
                for(int a = 0; a < A; ++a)
                    x[a] = pk::mul(x[a], __ldg(w + a * TN));
            }
        }
        else
        {
            const pk::c64 *w = reinterpret_cast<const pk::c64 *>(window2) + tid;
            const pk::c64 *t0 = reinterpret_cast<const pk::c64 *>(tw.tw0) + tid;
#pragma unroll
            for(int a = 0; a < P / 2; ++a)
            {
                pk::c64 lo = pk::from(v[a]), hi = pk::from(v[a + P / 2]);
                nzbits |= lo | hi;
                if(window2 != nullptr)
                {
                    lo = pk::mul(lo, __ldg(w + a * TN));
                    hi = pk::mul(hi, __ldg(w + (a + P / 2) * TN));
                }
                x[a] = pk::add(lo, hi);
                x[a + P / 2] = pk::cmul(pk::sub(lo, hi), __ldg(t0 + a * TN));
            }
        }
        return (nzbits & 0x7fffffff7fffffffull) != 0ull;
    }

    // The three passes.  Work buffer `buf` (L1 then L2); the natural-order result goes to out[k * OS] — `out` may be
    // the work buffer itself (OS = 1, ALIAS) or another array (the split plan interleaves two sub-FFTs with OS = 2).
    // nz_thread: this thread saw a non-zero sample; returns the block-wide OR (folded into the first barrier).
    template<int OS, bool ALIAS>
    static __device__ __forceinline__ bool run_core(pk::c64 (&x)[P], float2 *buf, const Tw3 &tw, int tid, bool nz_thread,
                                                    pk::c64 *out)
    {
        pk::c64 *b64 = reinterpret_cast<pk::c64 *>(buf);
        bool nz;
        // ---- pass 1: DFT over a (stride BC), twiddle W_M^(tid*ka), store L1[ka][b][c] at tid + ka*S1 ----
        pk::dft_bitrev<A>(x);
        {
            const pk::c64 *t1 = reinterpret_cast<const pk::c64 *>(tw.tw1) + tid;
            nz = __syncthreads_or(nz_thread ? 1 : 0) != 0; // previous users of the buffer are done
#pragma unroll
            for(int ka = 0; ka < A; ++ka)
            {
                pk::c64 y = x[bitrev<A>(ka)];
                if(ka > 0)
                    y = pk::cmul(y, __ldg(t1 + ka * TN));
                b64[tid + ka * G::S1] = y;
            }
        }
        __syncthreads();
        // ---- pass 2: lines (ka, c), c fastest; line l = tid + q*TN -> ka = tid/C + q*B, c = tid%C ----
        {
            const int c = tid % C;
            const pk::c64 *src = b64 + (tid / C) * G::S1 + c;
#pragma unroll
            for(int q = 0; q < G::LB; ++q)
#pragma unroll
                for(int b = 0; b < B; ++b)
                    x[q * B + b] = src[q * B * G::S1 + b * C];
            __syncthreads(); // L1 fully read before L2 (same memory) is written
            const pk::c64 *t2 = reinterpret_cast<const pk::c64 *>(tw.tw2) + c;
            pk::c64 *dst = b64 + (tid / C) * G::SA + c;
#pragma unroll
            for(int q = 0; q < G::LB; ++q)
            {
                pk::c64 y[B];
#pragma unroll
                for(int b = 0; b < B; ++b)
                    y[b] = x[q * B + b];
                pk::dft_bitrev<B>(y);
#pragma unroll
                for(int kb = 0; kb < B; ++kb)
                {
                    pk::c64 z = y[bitrev<B>(kb)];
                    if(kb > 0)
                        z = pk::cmul(z, __ldg(t2 + kb * C));
                    dst[q * B * G::SA + kb * G::SB] = z; // L2[kb][ka][c]
                }
            }
        }
        __syncthreads();
        // ---- pass 3: lines (ka, kb), ka fastest; line l = tid + q*TN -> ka = tid%A, kb = tid/A + q*TN/A ----
        {
            const pk::c64 *src = b64 + (tid / A) * G::SB + (tid % A) * G::SA;
#pragma unroll
            for(int q = 0; q < G::LC; ++q)
#pragma unroll
                for(int c = 0; c < C; ++c)
                    x[q * C + c] = src[q * (TN / A) * G::SB + c];
            if(ALIAS)
                __syncthreads(); // L2 fully read before X (same memory) is written
#pragma unroll
            for(int q = 0; q < G::LC; ++q)
            {
                pk::c64 y[C];
#pragma unroll
                for(int c = 0; c < C; ++c)
                    y[c] = x[q * C + c];
                pk::dft_bitrev<C>(y);
#pragma unroll
                for(int kc = 0; kc < C; ++kc)
                    out[(tid + q * TN + kc * (A * B)) * OS] = y[bitrev<C>(kc)]; // X[ka + A*kb + AB*kc]
            }
        }
        if(ALIAS)
            __syncthreads();
        return nz;
    }
    // v[a] windowed in x on entry; on exit X[k] sits in buf[k] (natural order)
    static __device__ __forceinline__ bool run(pk::c64 (&x)[P], float2 *buf, const Tw3 &tw, int tid, bool nz_thread)
    {
        if constexpr(!G::SPLIT2)
            return run_core<1, true>(x, buf, tw, tid, nz_thread, reinterpret_cast<pk::c64 *>(buf));
        else
        {
            // radix-2 decimation in frequency: y0 = lo + hi -> even bins, y1 = (lo - hi) W_M^n -> odd bins; each half is a
            // 4096-point FFT with exactly the 8192 plan's input layout (v[a] = y[a*256 + tid])
            using H = Fft3<N / 2>;
            pk::c64 *X = reinterpret_cast<pk::c64 *>(buf);
            float2 *work = buf + M;
            pk::c64 y0[P / 2], y1[P / 2];
#pragma unroll
            for(int a = 0; a < P / 2; ++a)
            {
                y0[a] = x[a];         // the radix-2 stage happened in finish_load
                y1[a] = x[a + P / 2];
            }
            const bool nz = H::template run_core<2, false>(y0, work, tw, tid, nz_thread, X);
            H::template run_core<2, false>(y1, work, tw, tid, false, X + 1);
            __syncthreads(); // X complete
            return nz;
        }
    }
};

} // namespace v3

// EXTRA: 0 = plain, 1 = + per-tick peak output (BASELINE config 5), 3 = + slope / fast peaks / skip mask / volume
// normalisation / roll-off as well.  Keeping the peak apart matters: ncu on config 5 (profiles/r01m_v3_c5.txt) showed the
// all-features epilogue costing 54 warp-instructions per bin although only the peak was in use.
template<int N, int CC, int R, int EXTRA, typename TS>
__global__ void __launch_bounds__(v3::Geo3<N>::TN, v3::Geo3<N>::MINB)
    stft_v3_kernel(const __grid_constant__ KParams p, const __grid_constant__ v3::Tw3 tw)
{
    using G = v3::Geo3<N>;
    using F = v3::Fft3<N>;
    constexpr int M = G::M, B = G::M, TN = G::TN, P = G::P;
    constexpr int HP = P / 2;      // pairs (k, M-k) per thread
    constexpr int SLICE = B / R;   // bins owned by one CTA
    constexpr int SP = SLICE / TN; // bins owned by one thread
    static_assert(SP >= 1 && SP * TN * R == B, "cluster size does not tile the bins");

    constexpr bool XP = (EXTRA & 1) != 0; // peak output
    constexpr bool XF = (EXTRA & 2) != 0; // slope, fast peaks, skip mask, volume normalisation, roll-off
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);
    constexpr bool DBUF = (R > 1) && v3::dbuf_inbox<N>();
    // [parity][R][CC][SLICE] linear magnitudes: own array (DBUF) or the FFT buffer itself (after barrier A)
    float *inbox0 = DBUF ? reinterpret_cast<float *>(buf + G::BUF) : reinterpret_cast<float *>(smem_raw);
    float *dbfull = reinterpret_cast<float *>(buf + G::BUF) + (DBUF ? 2 * CC * B : 0); // [dch][B] dB spectrum of MY tick
    float *pts = dbfull + (size_t)p.dch * B;
    __shared__ float red_scratch[2 * TN];
    __shared__ unsigned nzf[2][R];
    __shared__ unsigned redf[2][R];

    const int tid = threadIdx.x;
    const unsigned r = (R > 1) ? cluster_ctarank() : 0u;
    const int s = blockIdx.x / R;
    const int T = p.n_frames;
    const int dch = p.dch, och = p.och;
    const bool stereo = p.stereo != 0;
    const bool want_points = (p.out_points != nullptr) || (p.out_pixels != nullptr) || (p.out_min != nullptr);
    const bool mirror_each_frame = (p.out_db == nullptr) && p.write_hold;
    if constexpr(R > 1)
    {
        // distributed shared memory may only be addressed once every CTA of the cluster has started executing
        cluster_arrive();
        cluster_wait();
    }
    const uint32_t inbox_sa0 = smem_u32(inbox0);
    const uint32_t dbfull_sa = smem_u32(dbfull);

    // Bin bookkeeping.  Phase 1 produces, per thread, the pairs j < HP:  k1 = tid + j*TN  and  k2 = M - k1
    // (thread 0, j = 0: k2 := M/2, the self-paired bin; bin M itself does not exist).
    // R == 1: the EMA runs directly on those registers, state index i = 2*j (+1 for k2).
    // R  > 1: a thread owns bins r*SLICE + tid + i*TN, i < SP, fed through the inbox.
    const int k2_first = (tid == 0) ? M / 2 : M - tid; // partner of k1 = tid (pair j = 0)
    const int k2_base = M - tid;                      // partner of k1 = tid + j*TN is k2_base - j*TN for j >= 1
    auto bin_of = [&](int i) -> int {
        if constexpr(R == 1)
        {
            const int j = i >> 1;
            if((i & 1) == 0)
                return tid + j * TN;
            return (j == 0) ? k2_first : k2_base - j * TN;
        }
        else
            return (int)r * SLICE + tid + i * TN;
    };
    constexpr int NST = (R == 1) ? P : SP;

    float st[CC][NST];
    {
        const float *sp = p.state + (size_t)s * CC * B;
#pragma unroll
        for(int c = 0; c < CC; ++c)
#pragma unroll
            for(int i = 0; i < NST; ++i)
                st[c][i] = sp[c * B + bin_of(i)];
    }
    const unsigned char fl = p.flags[s];
    bool last_silent = (fl & 1u) != 0;
    bool po0 = (fl & 2u) != 0, po1 = (fl & 4u) != 0;
    bool po_valid = true;
    bool part0 = true, part1 = true;
    unsigned red_par = 0;

    const TS *pcm_s = Pcm<TS>::base(p.pcm) + (size_t)s * p.stream_stride;
    float *hold_s = p.hold_db + (size_t)s * och * B;

    // cluster-wide AND of the per-thread partial "outputs <= floor-10" flags of the last tick that produced outputs
    auto ensure_po_valid = [&]() {
        if(po_valid)
            return;
        const int a0 = __syncthreads_and(part0 ? 1 : 0);
        const int a1 = __syncthreads_and(part1 ? 1 : 0);
        if constexpr(R > 1)
        {
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
        }
        else
        {
            po0 = a0 != 0;
            if(dch > 1)
                po1 = a1 != 0;
        }
        po_valid = true;
    };

    // ---- pieces shared by the R == 1 and R > 1 flows -------------------------------------------------------------
    // gate of one capture channel for one tick, src/source_generic.cpp:63-95; returns "this channel is processed"
    auto gate_channel = [&](int c, bool nz_c, bool skip_all, const bool (&proc)[2], unsigned &silent_channels) -> bool {
        bool do_proc = !skip_all;
        if(!skip_all)
        {
            const bool silent = !nz_c;
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
        return do_proc;
    };
    // EMA of one bin, src/source_generic.cpp:124-132
    // (without temporal smoothing the engine passes g = 0, g2 = 1: 0*old + 1*mag == mag exactly, no branch needed)
    float ema_g = p.g, ema_g2 = p.g2; // per tick when the batch carries a gravity table (set_gravity below)
    auto set_gravity = [&](int t) {
        if(XF && p.g_tab != nullptr)
        {
            const float2 gt = __ldg(p.g_tab + t);
            ema_g = gt.x;
            ema_g2 = gt.y;
        }
    };
    auto ema = [&](float mag, float &state) {
        float oldval = state;
        if(XF && p.fast_peaks)
            oldval = fmaxf(mag, oldval);
        state = __fmaf_rn(ema_g, oldval, __fmul_rn(ema_g2, mag)); // one fused rounding, see the R == 1 flow
    };
    // split pass of pair j of my tick -> (|X[k1]|, |X[k2]|), normalised, slope applied (src/source_generic.cpp:110-122)
    auto split_pair = [&](const pk::c64 *X, const pk::c64 *twp, int j, float &m1, float &m2) {
        // |X| through MUFU.SQRT in its flush-to-zero form, as wf_fast2048.cuh: the subnormal-safe variant costs an FSETP and two
        // FMULs per bin (ncu, profiles/r01k_v3_8192.txt: 776 FMUL + 520 FSETP per N=8192 frame); powers below FLT_MIN
        // (|X| < 1e-19, -380 dBFS — digital silence) become exact zeros, which dbfs reports as DB_MIN.
        const int k1 = tid + j * TN;
        const pk::c64 a = X[k1];
        // X[M - k1]: descending addresses (conflict free); thread 0 pairs bin 0 with itself
        const pk::c64 bq = X[(j == 0 && tid == 0) ? 0 : (M - k1)];
        const pk::c64 b = pk::conj(bq);
        const pk::c64 sum = pk::add(a, b);
        const pk::c64 o = pk::mul_neg_i(pk::sub(a, b));
        const pk::c64 wo = pk::cmul(o, __ldg(twp + j * TN));
        const pk::c64 y1 = pk::add(sum, wo);
        const pk::c64 y2 = pk::sub(sum, wo);
        const pk::c64 s1 = pk::mul(y1, y1), s2 = pk::mul(y2, y2);
        float p1 = pk::re(s1) + pk::im(s1);
        float p2 = pk::re(s2) + pk::im(s2);
        if(j == 0)
        {
            // thread 0: second slot = bin M/2, whose split pass is 2*conj(X[M/2])
            const pk::c64 xm = X[M / 2];
            const pk::c64 sq = pk::mul(xm, xm);
            const float pm = 4.0f * (pk::re(sq) + pk::im(sq));
            p2 = (tid == 0) ? pm : p2;
        }
        pk::c64 m = pk::mul(pk::make(sqrt_approx_ftz(p1), sqrt_approx_ftz(p2)), pk::make(p.coef_half, p.coef_half));
        if(XF && p.slope != nullptr)
            m = pk::mul(m, pk::make(__ldg(p.slope + k1), __ldg(p.slope + ((j == 0) ? k2_first : k2_base - j * TN))));
        pk::split(m, m1, m2);
    };
    // outputs of one tick from the state registers, src/source_generic.cpp:136-179
    auto do_outputs = [&](int t, int f, const bool (&proc)[2]) {
        const float *prev_db = (p.out_db != nullptr && t > 0) ? p.out_db + ((size_t)s * T + (t - 1)) * dch * B : hold_s;
        float vc = 0.0f;
        if(XF && p.normalize)
        {
            const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + t] : 0.0f;
            vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
        }
        float *odb = (p.out_db != nullptr) ? p.out_db + ((size_t)s * T + t) * dch * B : nullptr;
        uint32_t gather_sa = 0u;
        if(R > 1 && want_points)
            gather_sa = mapa(dbfull_sa, (unsigned)f);
        float peak = -INFINITY;
        bool outs0 = true, outs1 = true;
        auto emit = [&](int d, int k, float outv, float &omax) {
            omax = fmaxf(omax, outv); // "all outputs <= floor-10" == !(max > floor-10)
            if(XP && k >= 1)
                peak = fmaxf(peak, outv);
            if(odb != nullptr)
                stg_stream(odb + d * B + k, outv);
            if(mirror_each_frame)
                hold_s[d * B + k] = outv;
            if(want_points)
            {
                if constexpr(R > 1)
                    st_cluster_f32(gather_sa + (uint32_t)((d * B + k) * sizeof(float)), outv);
                else
                    dbfull[d * B + k] = outv;
            }
        };
        auto finish = [&](float in, int k) -> float {
            // dbfs (src/source.hpp:293-299) as MUFU.LG2 + FMUL + FMNMX: lg2.approx.ftz(0) = -inf and lg2(x < 0) = NaN both
            // end up at DB_MIN = 20 log10(FLT_MIN) through the max (fmaxf drops a NaN); magnitudes below FLT_MIN (the
            // far tail of an EMA decay, < -758.6 dBFS) report DB_MIN instead of a value below it, as wf_fast2048.cuh.
            float outv = fmaxf(lg2_approx_ftz(in) * 6.02059991327962390f, p.db_min);
            if(XF && k >= 1)
            {
                if(p.normalize)
                    outv += vc; // :161-167
                if(p.rolloff != nullptr)
                    outv = fmaxf(outv - __ldg(p.rolloff + k), p.db_min); // :169-179
            }
            return outv;
        };
        const bool all_proc = proc[0] && (CC == 1 || proc[1]);
        if(R == 1 && CC == 1 && !XF && !last_silent && all_proc)
        {
            // hot path of the one-CTA-per-stream, one-channel kernel: dB of a bin pair with one packed multiply
            float omax = -INFINITY;
#pragma unroll
            for(int j = 0; j < NST / 2; ++j)
            {
                float d1, d2;
                pk::split(dbfs2(st[0][2 * j], st[0][2 * j + 1], p.db_min), d1, d2);
                emit(0, bin_of(2 * j), d1, omax);
                emit(0, bin_of(2 * j + 1), d2, omax);
            }
            outs0 = !(omax > p.floor_m10);
        }
        else if(!last_silent && all_proc)
        {
            // hot path: every channel processed this tick — straight-line code
            for(int d = 0; d < dch; ++d)
            {
                float omax = -INFINITY;
#pragma unroll
                for(int i = 0; i < NST; ++i)
                {
                    float in;
                    if(CC == 2 && !stereo)
                        in = (st[0][i] + st[CC - 1][i]) * 0.5f; // :150-154
                    else
                        in = (CC == 2 && d == 1) ? st[CC - 1][i] : st[0][i];
                    const int k = bin_of(i);
                    emit(d, k, finish(in, k), omax);
                }
                if(d == 0)
                    outs0 = !(omax > p.floor_m10);
                else
                    outs1 = !(omax > p.floor_m10);
            }
        }
        else
        {
            // rare paths: tick returned early (hold, :138-139) or a channel was skipped (stale dB re-converted)
            for(int d = 0; d < dch; ++d)
            {
                float omax = -INFINITY;
#pragma unroll 1
                for(int i = 0; i < NST; ++i)
                {
                    const int k = bin_of(i);
                    float s0 = 0.0f, s1 = 0.0f; // st[.][i] with a run-time i: select, no local-memory indexing
#pragma unroll
                    for(int ii = 0; ii < NST; ++ii)
                        if(ii == i)
                        {
                            s0 = st[0][ii];
                            s1 = st[CC - 1][ii];
                        }
                    float outv;
                    if(last_silent)
                        outv = prev_db[d * B + k];
                    else
                    {
                        float in;
                        if(CC == 2 && !stereo)
                        {
                            const float in0 = proc[0] ? s0 : prev_db[k];
                            in = (in0 + s1) * 0.5f;
                        }
                        else
                        {
                            const int c = (CC == 2) ? d : 0;
                            in = proc[c] ? ((c == 0) ? s0 : s1) : prev_db[c * B + k];
                        }
                        outv = finish(in, k);
                    }
                    emit(d, k, outv, omax);
                }
                if(d == 0)
                    outs0 = !(omax > p.floor_m10);
                else
                    outs1 = !(omax > p.floor_m10);
            }
        }
        if(!last_silent && p.gate)
        {
            part0 = outs0;
            part1 = outs1;
            po_valid = false;
        }
        if(p.out_silent != nullptr && r == 0 && tid == 0)
            p.out_silent[(size_t)s * T + t] = last_silent ? 1 : 0;
        if(XP && p.out_peak != nullptr)
        {
            const float gm = group_max<TN>(peak, red_scratch);
            if(tid == 0)
                atomic_max_float(p.out_peak + t, gm);
        }
    };

    // PCM prefetch: with 16 points per thread the NEXT frame's samples are requested as soon as the current ones have
    // been windowed (in flight during the whole FFT); with 32 there is no register room until the split pass is over.
    constexpr bool EARLY_PF = (P <= 16) && (CC == 1); // two capture channels: no register room either -> L2 prefetch
    // 32 points per thread: holding the next frame in 64 registers across a round makes ptxas spill them on arrival, so
    // the frame is only pulled into L2 ahead of time and loaded where it is consumed.
    constexpr bool KEEP_V = (P <= 16);
    float2 v[P];
    if((int)r < T)
    {
        if(KEEP_V)
            F::load_raw(v, pcm_s + (size_t)r * p.hop, p.aligned8, tid);
        else
            F::prefetch_l2(pcm_s + (size_t)r * p.hop, tid);
    }

    for(int t0 = 0; t0 < T; t0 += R)
    {
        const int nf = min(R, T - t0);
        const bool mine = (int)r < nf;
        const int my_t = t0 + (int)r;
        // next frame this CTA will need after (my tick, channel c)
        auto next_frame = [&](int c) -> const TS * {
            if(c + 1 < CC)
                return pcm_s + (size_t)(c + 1) * p.channel_stride + (size_t)my_t * p.hop;
            return (my_t + R < T) ? pcm_s + (size_t)(my_t + R) * p.hop : nullptr;
        };

        if constexpr(R == 1)
        {
            // ---- one CTA per stream: FFT -> gate -> split pass -> EMA per channel, all in registers ----
            const int t = t0;
            set_gravity(t);
            const bool skip_all = XF && (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + t] != 0);
            bool proc[2] = {false, false};
            unsigned silent_channels = 0;
#pragma unroll
            for(int c = 0; c < CC; ++c)
            {
                pk::c64 x[P];
                const bool nzt = F::finish_load(x, v, p.window2, tid, tw);
                const TS *nx = next_frame(c);
                if(nx != nullptr)
                {
                    if(EARLY_PF)
                        F::load_raw(v, nx, p.aligned8, tid);
                    else
                        F::prefetch_l2(nx, tid);
                }
                const bool nz = F::run(x, buf, tw, tid, nzt);
                if(!EARLY_PF && nx != nullptr)
                    F::load_raw(v, nx, p.aligned8, tid);
                const bool do_proc = gate_channel(c, nz, skip_all, proc, silent_channels);
                proc[c] = do_proc;
                const pk::c64 *X = reinterpret_cast<const pk::c64 *>(buf);
                const pk::c64 *twp = reinterpret_cast<const pk::c64 *>(p.tw_post) + tid;
                if(do_proc) // block-uniform: a channel that is not processed keeps its state and needs no split pass
                {
#pragma unroll
                    for(int j = 0; j < HP; ++j)
                    {
                        float m1, m2;
                        split_pair(X, twp, j, m1, m2);
                        // EMA of the pair, packed: g*old + (g2*mag) with ONE fused rounding on the first product, as
                        // wf_fast2048.cuh and the reference's AVX2 path (src/source_avx2.cpp:154); the cluster flow's scalar
                        // ema() below uses the same form, so R = 1 and R > 1 stay bit-identical.
                        pk::c64 old = pk::make(st[c][2 * j], st[c][2 * j + 1]);
                        pk::c64 m = pk::make(m1, m2);
                        if(XF && p.fast_peaks)
                            old = pk::make(fmaxf(m1, st[c][2 * j]), fmaxf(m2, st[c][2 * j + 1]));
                        m = pk::fma(pk::make(ema_g, ema_g), old, pk::mul(pk::make(ema_g2, ema_g2), m));
                        pk::split(m, st[c][2 * j], st[c][2 * j + 1]);
                    }
                }
            }
            do_outputs(t, 0, proc);
            if(want_points)
            {
                __syncthreads();
                display_stage<TN>(p, dbfull, pts, B, dch, (size_t)s * T + t, tid, true, red_scratch);
            }
        }
        else
        {
            float magr[CC][P]; // [c][2*j] = |X[k1]|, [c][2*j+1] = |X[k2]|
            unsigned nzbits = 0;
            // ---- phase 1: window, FFT, split pass, magnitude of my tick (src/source_generic.cpp:97-122) ----
            if(mine)
            {
#pragma unroll
                for(int c = 0; c < CC; ++c)
                {
                    pk::c64 x[P];
                    if(!KEEP_V)
                        F::load_raw(v, pcm_s + (size_t)c * p.channel_stride + (size_t)my_t * p.hop, p.aligned8, tid);
                    const bool nzt = F::finish_load(x, v, p.window2, tid, tw);
                    const TS *nx = next_frame(c);
                    if(nx != nullptr)
                    {
                        if(EARLY_PF)
                            F::load_raw(v, nx, p.aligned8, tid);
                        else
                            F::prefetch_l2(nx, tid);
                    }
                    const bool nz = F::run(x, buf, tw, tid, nzt);
                    if(KEEP_V && !EARLY_PF && c + 1 < CC)
                        F::load_raw(v, nx, p.aligned8, tid); // the other channel of my tick
                    nzbits |= nz ? (1u << c) : 0u;
                    const pk::c64 *X = reinterpret_cast<const pk::c64 *>(buf);
                    const pk::c64 *twp = reinterpret_cast<const pk::c64 *>(p.tw_post) + tid;
#pragma unroll
                    for(int j = 0; j < HP; ++j)
                        split_pair(X, twp, j, magr[c][2 * j], magr[c][2 * j + 1]);
                }
            }
            const int par = DBUF ? ((t0 / R) & 1) : 0;
            const uint32_t inbox_sa = inbox_sa0 + (uint32_t)(par * CC * B * sizeof(float));
            const float *inbox = inbox0 + par * CC * B;
            if constexpr(!DBUF)
            {
                __syncthreads(); // my FFT buffer is free: it becomes the inbox
                cluster_arrive(); // barrier A
                cluster_wait();
            }
            // (DBUF: inbox[par] was last read two rounds ago, before every peer arrived at the previous round's barrier)
            // ---- phase 2: all-to-all through distributed shared memory ----
            if(mine)
            {
                // blocks of TN bins: k1 lies in block j, k2 in block P-1-j (thread 0: k2 = M - j*TN opens block P-j, or M/2)
                const int t0off = (tid == 0) ? 0 : TN - tid;
#pragma unroll
                for(int c = 0; c < CC; ++c)
#pragma unroll
                    for(int j = 0; j < HP; ++j)
                    {
                        const uint32_t d1 = mapa(inbox_sa, (unsigned)(j / SP)) +
                                            (uint32_t)(((r * CC + c) * SLICE + tid + (j % SP) * TN) * sizeof(float));
                        st_cluster_f32(d1, magr[c][2 * j]);
                        const int blk = (tid == 0) ? ((j == 0) ? HP : P - j) : (P - 1 - j);
                        const uint32_t d2 = mapa(inbox_sa, (unsigned)(blk / SP)) +
                                            (uint32_t)(((r * CC + c) * SLICE + t0off + (blk % SP) * TN) * sizeof(float));
                        st_cluster_f32(d2, magr[c][2 * j + 1]);
                    }
                if(tid < R)
                    st_cluster_u32(mapa(smem_u32(&nzf[par][r]), (unsigned)tid), nzbits);
            }
            cluster_arrive(); // barrier B
            if(KEEP_V && !EARLY_PF && mine && my_t + R < T)
                F::load_raw(v, pcm_s + (size_t)(my_t + R) * p.hop, p.aligned8, tid);
            cluster_wait();

            // ---- phase 3: my bins through the round's ticks, in order ----
            for(int f = 0; f < nf; ++f)
            {
                const int t = t0 + f;
                set_gravity(t);
                const unsigned nzb = nzf[par][f];
                const bool skip_all = XF && (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + t] != 0);
                bool proc[2] = {false, false};
                unsigned silent_channels = 0;
#pragma unroll
                for(int c = 0; c < CC; ++c)
                {
                    const bool do_proc = gate_channel(c, ((nzb >> c) & 1u) != 0, skip_all, proc, silent_channels);
                    proc[c] = do_proc;
                    if(do_proc) // cluster-uniform: an unprocessed channel keeps its state
                    {
#pragma unroll
                        for(int i = 0; i < NST; ++i)
                            ema(inbox[(f * CC + c) * SLICE + tid + i * TN], st[c][i]);
                    }
                }
                do_outputs(t, f, proc);
            }
            // ---- phase 4: render-time stages of my tick from the gathered dB spectrum ----
            if(want_points)
            {
                cluster_arrive(); // barrier C
                cluster_wait();
                if(mine)
                    display_stage<TN>(p, dbfull, pts, B, dch, (size_t)s * T + my_t, tid, true, red_scratch);
            }
        }
        // (the next round's FFT starts with a block barrier before it overwrites the buffer)
    }

    // ---- state back to the engine (my bins) ----
    ensure_po_valid();
    {
        float *sp = p.state + (size_t)s * CC * B;
#pragma unroll
        for(int c = 0; c < CC; ++c)
#pragma unroll
            for(int i = 0; i < NST; ++i)
                sp[c * B + bin_of(i)] = st[c][i];
        if(p.write_hold && p.out_db != nullptr && T > 0)
        {
            const float *last = p.out_db + ((size_t)s * T + (T - 1)) * dch * B;
            for(int d = 0; d < dch; ++d)
#pragma unroll
                for(int i = 0; i < NST; ++i)
                    hold_s[d * B + bin_of(i)] = last[d * B + bin_of(i)];
        }
        if(CC == 2 && !stereo && p.write_hold)
        {
#pragma unroll
            for(int i = 0; i < NST; ++i)
                hold_s[B + bin_of(i)] = st[1][i];
        }
        if(r == 0 && tid == 0)
            p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (po0 ? 2u : 0u) | (po1 ? 4u : 0u));
    }
    if constexpr(R > 1)
    {
        cluster_arrive(); // no CTA may exit while a peer can still address its shared memory
        cluster_wait();
    }
}

} // namespace wf
