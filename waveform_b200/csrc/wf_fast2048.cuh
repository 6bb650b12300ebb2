// wf_fast2048.cuh — hand-specialised sm_90a kernel for the headline shape: N = 2048, one capture
// channel, 16-byte aligned frames (hop % 4 == 0), spectrum output only.
//
// One WARP owns one stream and walks its frames; per frame:
//   * the 8 KB PCM frame is staged HBM -> shared memory by a TMA bulk copy (cp.async.bulk + mbarrier),
//     issued one frame ahead (during the previous frame's epilogue) so the warp never waits on DRAM;
//   * the packed 1024-point complex FFT is two radix-32 register passes (32 points per lane) with ONE
//     padded shared-memory transpose between them (conflict-free 64-bit accesses);
//   * the real-FFT split pass processes bins k and N/2-k TOGETHER (one twiddle multiply for two bins),
//     after a half-size exchange so that each lane owns both bins of its 16 pairs;
//   * |X| via MUFU.SQRT, EMA with state in registers across the stream's frames, dB via MUFU.LG2,
//     32 coalesced 128-byte store instructions per frame.
// Tables (window, inter-pass twiddles, split twiddles: 20 KB) live in shared memory once per CTA.
//
// Semantics are those of wf_kernels.cuh / src/source_generic.cpp:26-180; differences are confined to the
// last-ulp behaviour of sqrt/log (well inside the 1e-5 parity bar, see DESIGN.md §Parity).
#pragma once
#include "wf_kernels.cuh"

namespace wf {

namespace fast {

constexpr int kN = 2048;
constexpr int kM = 1024;
constexpr int kWarpBufBytes = 32 * 33 * 8; // padded transpose buffer, also the TMA landing zone (8192 B used)
constexpr int kStateBytes = 16 * 32 * 8; // EMA state of the stream: [pair q][lane] -> (bin k1, bin k2)
constexpr int kWarpBytes = kWarpBufBytes + kStateBytes + 16; // + mbarrier
constexpr int kTableBytes = (1024 + 1024 + 512) * 8;
constexpr int kMaxWarpsPerCta = 16; // 1 CTA/SM: 16 warps x 12.3 KB + 20 KB tables = 216 KB of shared memory
constexpr int smem_bytes(int warps_per_cta) { return kTableBytes + warps_per_cta * kWarpBytes; }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted on the mbarrier
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ float sqrt_approx(float x)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ float lg2_approx_ftz(float x)
{
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// dbfs (src/source.hpp:293-299) on the MUFU.LG2 path: 20 log10(m) = (20 log10 2) log2(m), two bins at a time.
// Magnitudes below FLT_MIN (digital silence, the far tail of an EMA decay: < -758.6 dBFS) report DB_MIN —
// the reference reports DB_MIN for exact zero and a value below DB_MIN for subnormals; this kernel clamps
// those to DB_MIN (the generic kernel keeps the exact behaviour).  See DESIGN.md §Parity.
__device__ __forceinline__ pk::c64 dbfs2(float m1, float m2, float db_min)
{
    constexpr float k = 6.02059991327962390f; // 20 log10(2)
    pk::c64 d = pk::mul(pk::make(lg2_approx_ftz(m1), lg2_approx_ftz(m2)), pk::make(k, k));
    // lg2.approx.ftz(x < FLT_MIN) = -inf and 20 log10(FLT_MIN) == DB_MIN, so the clamp is one max per bin
    float d1, d2;
    pk::split(d, d1, d2);
    return pk::make(fmaxf(d1, db_min), fmaxf(d2, db_min));
}

} // namespace fast

// One CTA per SM with up to MAXW warps (16 -> 128 registers/thread, 12 -> 168).  WIN is not a template
// parameter: without a window the shared "window" table simply holds the magnitude normalisation constant.
template<int MAXW, bool TSM, bool GATE, bool EXTRA>
__global__ void __launch_bounds__(MAXW * 32, 1) stft2048_fast_kernel(const __grid_constant__ KParams p)
{
    using namespace fast;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2 *s_win = reinterpret_cast<float2 *>(smem_raw);
    float2 *s_twA = s_win + 1024; // [k2][n1] = W_1024^(k2*n1)
    float2 *s_twP = s_twA + 1024; // [q][lane] = W_2048^(lane + 32 q), q < 16
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int warps_per_cta = blockDim.x >> 5;
    unsigned char *wbase = reinterpret_cast<unsigned char *>(s_twP + 512) + warp * kWarpBytes;
    float2 *buf = reinterpret_cast<float2 *>(wbase);
    float2 *sst = reinterpret_cast<float2 *>(wbase + kWarpBufBytes) + lane; // this lane's column of the state
    uint64_t *mbar = reinterpret_cast<uint64_t *>(wbase + kWarpBufBytes + kStateBytes);

    // ---- CTA prologue: tables -> shared, mbarriers ----
    // The window table carries the magnitude normalisation (2/sum(w))/2 so the epilogue needs no extra multiply.
    for(int i = threadIdx.x; i < 1024; i += blockDim.x)
    {
        {
            const float2 w = (p.window2 != nullptr) ? __ldg(p.window2 + i) : make_float2(1.0f, 1.0f);
            s_win[i] = make_float2(w.x * p.coef_half, w.y * p.coef_half);
        }
        s_twA[i] = __ldg(p.tw + (((i >> 5) * (i & 31)) & 1023));
        if(i < 512)
            s_twP[i] = __ldg(p.tw_post + i);
    }
    int *seg_done = reinterpret_cast<int *>(mbar + 1); // this warp's head segment is finished (split mode)
    if(lane == 0)
    {
        mbar_init(mbar, 1);
        *seg_done = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (tables, barriers) touches only immutable data and may overlap
    // the tail of the previous launch on this stream; per-stream state / PCM / outputs are touched only after the
    // previous grid has completed and flushed.  Let the next launch start its own prologue as early as possible.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // Streams are dealt round-robin to CTAs (= SMs) first and to the CTA's warps second, so every SM gets
    // n_streams/gridDim (+-1) streams whatever the warp count: stream of (cta c, local index i) = c + i*gridDim.
    const int S = p.n_streams, T = p.n_frames;
    const int G = gridDim.x;
    const int n_local = (S > (int)blockIdx.x) ? (S - (int)blockIdx.x + G - 1) / G : 0;
    constexpr int B = kM;
    uint32_t phase = 0;

    // bins owned by this lane: first output of pair q -> k1 = lane + 32 q; second -> k2 = kb + 32 (31 - q)
    const int jp = (32 - lane) & 31;
    const int kb = jp + (lane == 0 ? 32 : 0);
    const int k2_q0 = (lane == 0) ? 512 : (kb + 992);

    // ---- work list of this warp ----
    // Whole streams, dealt round-robin (local index li = warp, warp + W, ...), leave the last round partly empty: 4096 streams
    // are 27.7 per SM, i.e. 16 busy warps for one round and 11.7 for the second.  In split mode (p.split, at least one
    // stream per warp, more than one tick) the SM's n_local * T frames are cut into W equal runs of consecutive frames
    // instead: a warp's run is [tail of stream a][whole streams][head of stream b], and a stream is continued by the next
    // warp exactly as it would be by the next call (state, flags and mirror go through global memory).  Order inside a
    // warp: the head first (it depends on nothing), the whole streams, the tail last — by then warp - 1 has long finished
    // the head it started with; the hand-over is a shared-memory flag behind a CTA-scope fence.
    // (worth it only when the partly empty last round costs more than the hand-overs: the makespan shrinks by
    // (rounds * W - n_local) * T / W frame times, each of the W - 1 hand-overs adds a state round trip)
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
    const int full0 = (u0 + T - 1) / T, full1 = u1 / T; // whole streams [full0, full1)
    const int has_head = (split && (u1 % T) != 0) ? 1 : 0, has_tail = (split && (u0 % T) != 0) ? 1 : 0;
    const int nseg = split ? (has_head + max(full1 - full0, 0) + has_tail)
                           : ((n_local > warp) ? (n_local - warp + warps_per_cta - 1) / warps_per_cta : 0);
    // segment j -> (local stream index, first tick, end tick)
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
        mbar_expect_tx(mbar, kN * 4);
        tma_load_1d(buf, p.pcm + (size_t)(blockIdx.x + li * G) * p.stream_stride + (size_t)t0 * p.hop, kN * 4, mbar);
    }

    for(int j = 0; j < nseg; ++j)
    {
        int li, t0, t1;
        segment(j, li, t0, t1);
        const int s = (int)blockIdx.x + li * G;
        // the next segment (its first frame and state are prefetched under the last tick of this one)
        int s_next = -1, t0_next = 0;
        if(j + 1 < nseg)
        {
            int li2, t12;
            segment(j + 1, li2, t0_next, t12);
            s_next = (int)blockIdx.x + li2 * G;
        }
        if(t0 > 0)
        {
            // continuation of a stream whose first ticks the previous warp ran as its head segment
            // (atomics on the flag, fences around them: the hand-over is a release / acquire pair at CTA scope)
            int *prev_done = reinterpret_cast<int *>(wbase - kWarpBytes + kWarpBufBytes + kStateBytes + 8);
            if(lane == 0)
                while(atomicAdd(prev_done, 0) == 0)
                    ;
            __syncwarp();
            __threadfence_block();
        }
        // ---- per-stream state: global (natural bin order) -> shared ([pair][lane]) ----
        {
            const float *sp = p.state + (size_t)s * B;
#pragma unroll
            for(int q = 0; q < 16; ++q)
                sst[q * 32] = make_float2(sp[lane + 32 * q], sp[(q == 0) ? k2_q0 : (kb + 32 * (31 - q))]);
        }
        const unsigned char fl = p.flags[s];
        bool last_silent = (fl & 1u) != 0;
        bool prev_out_silent = (fl & 2u) != 0;
        // bit 3: the m_decibels mirror of this stream was NOT written by the previous call because it equals
        // dbfs(state) (see the end of this loop); it is rebuilt from the state wherever it is needed
        const bool hold_lazy = (fl & 8u) != 0;
        bool last_from_state = false; // the last tick's outputs are dbfs(state) (normal tick), not a hold / quirk
        const float *pcm_s = p.pcm + (size_t)s * p.stream_stride;
        float *hold_s = p.hold_db + (size_t)s * B;

#pragma unroll 1
        for(int t = t0; t < t1; ++t)
        {
            // ---- frame from shared (TMA-staged), window in the load prologue ----
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

            // ---- two radix-32 register passes (unrolled: a rolled loop costs ~70 register moves per frame at the
            //      back-edge, and the code still fits the instruction cache) ----
#pragma unroll
            for(int pass = 0; pass < 2; ++pass)
            {
                pk::dft_bitrev<32>(v);
                if(pass == 0)
                {
                    // inter-pass twiddle W_1024^(n1 k2), then transpose through the (padded) shared buffer
                    __syncwarp(); // every lane has read the frame before the buffer becomes the transpose area
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
                    __syncwarp(); // all generic-proxy accesses to buf are done: it can take the next frame
                    // the next stream's EMA state (4 KB, one 128-byte line per lane) is pulled into L2 now, so that the
                    // synchronous state load at the top of the stream loop does not pay DRAM latency (matters when a
                    // stream has few frames: the 65536 x 1 layout loads a state per frame)
                    if(t + 1 == t1 && s_next >= 0 && t0_next == 0)
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(p.state + (size_t)s_next * B + lane * 32));
                    // prefetch the next frame (or the next stream's first frame) under pass B + epilogue
                    if(lane == 0)
                    {
                        const float *next = nullptr;
                        if(t + 1 < t1)
                            next = pcm_s + (size_t)(t + 1) * p.hop;
                        else if(s_next >= 0)
                            next = p.pcm + (size_t)s_next * p.stream_stride + (size_t)t0_next * p.hop;
                        if(next != nullptr)
                        {
                            fence_proxy_async();
                            mbar_expect_tx(mbar, kN * 4);
                            tma_load_1d(buf, next, kN * 4, mbar);
                        }
                    }
                }
            }
            // now X[lane + 32 k1] = v[bitrev(k1)]

            // The split pass needs X[1024-k] next to X[k]: lane j fetches the upper half of lane (32-j)%32 by
            // warp shuffle (lane 0 pairs within its own registers, one index higher).
            // ---- gate (src/source_generic.cpp:63-95), single capture channel ----
            const bool skip_all = EXTRA && (p.skip_mask != nullptr) && (p.skip_mask[(size_t)s * T + t] != 0);
            bool do_proc = !skip_all;
            if(!skip_all)
            {
                if(nz)
                    last_silent = false;
                else if(GATE)
                {
                    if(last_silent)
                        do_proc = false;
                    else if(prev_out_silent)
                    {
                        last_silent = true; // ++silent_channels >= 1
                        do_proc = false;
                    }
                }
            }

            float *odb = p.out_db + ((size_t)s * T + t) * B;
            float vc = 0.0f;
            if(EXTRA && p.normalize)
            {
                const float rms = (p.input_rms != nullptr) ? p.input_rms[(size_t)s * T + t] : 0.0f;
                vc = fminf(p.vol_target - dbfs(rms, p.db_min), p.max_gain);
            }
            bool outs = true;
            float peak = -INFINITY;
            // gravity of this tick: the call's scalar, or (EXTRA variant only) the per-tick table of a TV-exponential batch
            const float2 gt = (EXTRA && p.g_tab != nullptr) ? __ldg(p.g_tab + t) : make_float2(p.g, p.g2);

            if(do_proc && !last_silent)
            {
                // ---- hot path: split pass -> |X| -> slope -> EMA -> dBFS -> (volume, roll-off) -> store ----
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
                        // lane 0: the pair (0, 1024) has no bin 1024; its second slot carries bin 512 = conj(X[512])
                        const pk::c64 x512 = v[bitrev<32>(16)];
                        const pk::c64 sq = pk::mul(x512, x512);
                        const float p512 = 4.0f * (pk::re(sq) + pk::im(sq));
                        p2 = (lane == 0) ? p512 : p2;
                    }
                    pk::c64 m = pk::make(sqrt_approx(p1), sqrt_approx(p2)); // (|X[k1]|, |X[k2]|), normalised via the window
                    if(EXTRA && p.slope != nullptr)
                        m = pk::mul(m, pk::make(__ldg(p.slope + k1), __ldg(p.slope + k2)));
                    pk::c64 *sst64 = reinterpret_cast<pk::c64 *>(sst);
                    if(TSM)
                    {
                        pk::c64 old = sst64[q * 32];
                        if(EXTRA && p.fast_peaks)
                            old = pk::make(fmaxf(pk::re(m), pk::re(old)), fmaxf(pk::im(m), pk::im(old)));
                        // g*old + g2*new with one fused rounding, as the reference's AVX2 path (src/source_avx2.cpp:154)
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
                            d2 = fmaxf(d2 - __ldg(p.rolloff + k2), p.db_min);
                        }
                        if(k1 >= 1)
                            peak = fmaxf(peak, d1);
                        peak = fmaxf(peak, d2);
                    }
                    if(GATE)
                        outs &= !(d1 > p.floor_m10) & !(d2 > p.floor_m10);
                    stg_stream(odb + k1, d1);
                    stg_stream(odb + k2, d2);
                }
                last_from_state = true;
            }
            else
            {
                // ---- rare path: tick returned early (hold, src/source_generic.cpp:138-139) or the channel was
                //      skipped while the tick went on (stale dB re-converted, SURVEY appendix A quirk) ----
                // Previous outputs: the row of tick t-1, or (t == 0) the engine's m_decibels mirror — which the previous
                // call may have left implicit (hold_lazy: it is dbfs(state), and the state is in shared memory).
                const float *prev_db = (t > 0) ? (odb - B) : hold_s;
                const bool from_state = (t == 0) && hold_lazy;
#pragma unroll 1
                for(int q = 0; q < 16; ++q)
                {
                    const int k1 = lane + 32 * q;
                    const int k2 = (q == 0) ? k2_q0 : (kb + 32 * (31 - q));
                    float o1, o2;
                    if(from_state)
                    {
                        const float2 stv = sst[q * 32];
                        pk::split(dbfs2(stv.x, stv.y, p.db_min), o1, o2);
                    }
                    else
                    {
                        o1 = prev_db[k1];
                        o2 = prev_db[k2];
                    }
                    if(!last_silent)
                    {
                        o1 = dbfs(o1, p.db_min);
                        o2 = dbfs(o2, p.db_min);
                        if(EXTRA)
                        {
                            if(p.normalize)
                            {
                                if(k1 >= 1)
                                    o1 += vc;
                                o2 += vc;
                            }
                            if(p.rolloff != nullptr)
                            {
                                if(k1 >= 1)
                                    o1 = fmaxf(o1 - __ldg(p.rolloff + k1), p.db_min);
                                o2 = fmaxf(o2 - __ldg(p.rolloff + k2), p.db_min);
                            }
                        }
                    }
                    outs &= !(o1 > p.floor_m10) & !(o2 > p.floor_m10);
                    if(k1 >= 1)
                        peak = fmaxf(peak, o1);
                    peak = fmaxf(peak, o2);
                    odb[k1] = o1;
                    odb[k2] = o2;
                }
                last_from_state = false;
            }
            if(GATE && !last_silent)
                prev_out_silent = __all_sync(0xffffffffu, outs);
            if(p.out_silent != nullptr && lane == 0)
                p.out_silent[(size_t)s * T + t] = last_silent ? 1 : 0;
            if(EXTRA)
            {
                if(p.out_peak != nullptr)
                {
                    const float gm = group_max<32>(peak, nullptr);
                    if(lane == 0)
                        atomic_max_float(p.out_peak + t, gm);
                }
            }
        }

        // ---- state back to the engine; m_decibels mirror for the next call's gate / hold paths ----
        {
            float *sp = p.state + (size_t)s * B;
            const float *last = p.out_db + ((size_t)s * T + (t1 - 1)) * B;
            const bool plain = !EXTRA || (!p.normalize && p.rolloff == nullptr);
            // The mirror equals dbfs(state) after a normal tick without volume / roll-off post-processing: do not spend
            // 4 KB of HBM writes per stream on it, set bit 3 instead (the engine materialises it on demand, see
            // materialize_hold_kernel; this kernel rebuilds it from the state in its rare path).
            const bool lazy = last_from_state && plain && (p.lazy_hold != 0);
#pragma unroll
            for(int q = 0; q < 16; ++q)
            {
                const int k1 = lane + 32 * q;
                const int k2 = (q == 0) ? k2_q0 : (kb + 32 * (31 - q));
                const float2 stv = sst[q * 32];
                sp[k1] = stv.x;
                sp[k2] = stv.y;
                if(p.write_hold && !lazy)
                {
                    if(last_from_state && plain)
                    {
                        float h1, h2;
                        pk::split(dbfs2(stv.x, stv.y, p.db_min), h1, h2); // identical to what the last tick stored
                        hold_s[k1] = h1;
                        hold_s[k2] = h2;
                    }
                    else
                    {
                        hold_s[k1] = last[k1];
                        hold_s[k2] = last[k2];
                    }
                }
            }
            if(lane == 0)
                p.flags[s] = (unsigned char)((last_silent ? 1u : 0u) | (prev_out_silent ? 2u : 0u) | 4u | (lazy ? 8u : 0u));
        }
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
