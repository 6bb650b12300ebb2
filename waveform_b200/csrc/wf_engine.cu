// wf_engine.cu — libwfstft.so: the C ABI of include/wfstft.h on top of the fused sm_90a kernel.
//
// Host responsibilities (mirrors what WAVSource owns in the reference, src/source.hpp:95-347):
//   * settings -> tables (wf_tables.cpp ≙ WAVSource::update), uploaded once per engine
//   * per-stream recurrence state in device memory (m_tsmooth_buf, m_decibels, m_last_silent)
//   * staging of host buffers, kernel dispatch by (fft_size, capture_channels), error reporting
// There is no CPU compute path: if CUDA is unavailable wf_create fails.
#include <cuda_runtime.h>

#include <cmath>
#include <algorithm>
#include <array>
#include <cstdio>
#include <utility>
#include <cstring>
#include <string>
#include <vector>

#include "wf_host.hpp"
#include "wf_kparams.hpp"
#include "wf_anyn.hpp"
#include "wf_fast2048.hpp"
#include "wf_fused.hpp"
#include "wf_wide.hpp"
#include "wf_v3.hpp"
#include "wf_team2048.hpp"
#include "wf_warp2.hpp"
#include "wf_par16384.hpp"
#include "wf_render.hpp"
#include "wf_sm90.cuh"
#include "wf_splice.hpp"
#include "wf_nvtx.hpp"
#include "wf_tables.hpp"
#include "wfstft.h"

using namespace wf;

// Environment knobs of the spectrum engine, read at wf_create: A/B switches for tests and tools.  None changes a result.
struct SpectrumKnobs {
    bool force_generic = env_flag("WF_FORCE_GENERIC", false); // bypass the specialised N=2048 kernels
    bool v3 = env_flag("WF_V3", true);             // 0: the first-generation kernels instead of the CTA-per-tick kernel
    int wide_r = env_int("WF_WIDE_R", 0);          // 1|2|4|8: cluster size of the wide and CTA-per-tick kernels (1 = no
                                                   // wide kernel); 0 = automatic
    int team_w = env_int("WF_TEAM_W", 0);          // 4|8|16: team size of wf_team2048.cuh; 1 = never a team; 0 = automatic
    bool par16384 = env_flag("WF_PAR16384", true); // 0: N=16384 stays on the CTA-per-tick kernel
    bool warp2 = env_flag("WF_WARP2", true);       // 0: non-power-of-two sizes stay on the any-N kernel
    bool warp2_display = env_flag("WF_WARP2_DISPLAY", true); // 0: display outputs stay on the CTA-per-tick / any-N kernels
    bool split = env_flag("WF_SPLIT", true);       // 0: whole streams per warp in the N=2048 warp-per-stream kernel
    bool zero_copy = env_flag("WF_ZERO_COPY", true); // 0: always stage host buffers through device memory
};

struct wf_engine : HostCore {
    Tables tab;
    std::string last_kernel;    // name of the spectrum kernel the most recent launch_range dispatched to (wf_last_kernel_name)
    bool hold_implicit = false; // some stream may carry flags bit 3 (m_decibels mirror left implicit by the N=2048 kernels)
    bool hold_replayed = false; // an N=2048 kernel was captured: any replay may set bit 3, so hold_implicit stays set
    SpectrumKnobs knobs;
    Warp2Plan warp2;            // compiled warp-per-stream plan of this fft size (L == 0: none)
    AnyPlan any{};              // run-time plan of the any-N kernel (sizes without a templated kernel)

    // device tables
    DevBuf<float> d_window, d_slope, d_rolloff, d_tw, d_tw_post;
    DevBuf<float> d_tw1, d_tw2, d_tw0; // inter-pass twiddles of the CTA-per-tick kernel (wf_v3.cuh), N = 4096/8192/16384
    DevBuf<float> d_interp_idx, d_interp_w, d_gauss;
    DevBuf<int> d_band_widths, d_band_offsets;
    // per-stream state
    DevBuf<float> d_state, d_hold;
    DevBuf<unsigned char> d_flags;
    DevBuf<float> d_ring; // [max_streams][capture_channels][N + D] capture rings (wf_batch.capture_ring), allocated on first use
    int D = 0;            // samples the audio sync offset holds back (wf_config.sync_offset_ms; 0 without one)
    // [max_streams] samples each ring slot still needs before its first real tick (D at creation): counted down on the
    // device by the splice kernel (d_owed), and on the host by eager calls (owed).  Replays only lower the device's counts,
    // so owed[s] == 0 means the device's count is 0 too; only then does a ring call go without the start-up mask.
    DevBuf<long long> d_owed;
    std::vector<long long> owed;
    bool startup = false;         // the current ring call may still have start-up ticks (some owed > 0)
    DevBuf<unsigned char> s_mask; // [n_streams][n_frames] start-up ticks ORed with the caller's skip_mask
    // staging for host-pointer batches (grown on demand); each counts floats whatever it holds (int16 PCM, skip_mask and
    // out_silent bytes), so that batch_bufs can name any of them
    DevBuf<float> s_pcm, s_out_db, s_out_points, s_rms, s_skip, s_silent, s_peak, s_px, s_min;
    DevBuf<float> s_gtab; // [n_frames][2] per-tick (g, 1-g) of a TV-exponential batch with frame_seconds
    std::vector<float> h_gtab;
    DevBuf<float> s_scratch; // any-N kernel work buffers when N/2 complex points x 2 exceed shared memory
    DevBuf<float> s_render;  // wf_render: one dB row per group when a row does not fit in shared memory
    DevBuf<float> s_window;  // frames of a ring call in the plain layout, in the call's sample type (counts floats, as s_pcm)
    DevBuf<unsigned char> s_state; // staging of wf_get_state / wf_set_state (StateSections)
    std::vector<unsigned char> h_state;
    // zero-copy verdict of the last host-pointer batch (live ticks reuse the same buffers every call): pcm, then the
    // buffers of batch_bufs
    static constexpr int kBatchBufs = 8;
    const void *zc_ptrs[1 + kBatchBufs] = {};
    bool zc_ok = false, zc_dev = false, zc_valid = false;
    // copy/compute pipeline for host-pointer batches
    static constexpr int kMaxChunks = 16;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t chunk_in[kMaxChunks] = {}, chunk_k[kMaxChunks] = {}, ev_fork = nullptr, ev_join = nullptr;
};

// The engine's maintenance kernels (only this unit launches them).
namespace wf {

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
            const float l = lg2_approx_ftz(state[(size_t)s * B + k]);
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

// wf_get_state / wf_set_state, one CTA per stream of [0, count) (the device arrays start at the first): the state to or from
// the staging sections x_* (null = skipped).  Restored hold rows set the display bits the kernels keep, and flags bit 0.
template<bool SET>
static __device__ void copy_section(float *dev, float *x, long long off, long long n)
{
    for(long long k = off + threadIdx.x; x && k < off + n; k += blockDim.x)
        (SET ? dev[k] : x[k]) = (SET ? x[k] : dev[k]);
}
template<bool SET>
static __global__ void spectrum_state_kernel(float *state, float *hold, unsigned char *flags, float *x_tsmooth, float *x_hold,
                                             unsigned char *x_flags, int count, int cc, int och, int dch, int B, float thr)
{
    const long long ts = (long long)cc * B, hs = (long long)och * B;
    for(int i = blockIdx.x; i < count; i += gridDim.x)
    {
        copy_section<SET>(state, x_tsmooth, i * ts, ts);
        copy_section<SET>(hold, x_hold, i * hs, hs);
        unsigned bits = (dch == 1) ? 4u : 0u;
        for(int d = 0; SET && x_hold && d < dch; ++d)
        {
            bool above = false;
            for(int k = threadIdx.x; k < B; k += blockDim.x)
                above |= x_hold[i * hs + (long long)d * B + k] > thr;
            bits |= __syncthreads_or(above) ? 0u : 2u << d; // every bin of row d <= floor_db - 10
        }
        if(threadIdx.x == 0 && !SET && x_flags)
            x_flags[i] = flags[i] & 1u;
        if(threadIdx.x == 0 && SET && x_hold)
            flags[i] = (unsigned char)((flags[i] & 1u) | bits);
        if(threadIdx.x == 0 && SET && x_flags)
            flags[i] = (unsigned char)((flags[i] & ~1u) | (x_flags[i] & 1u));
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

} // namespace wf

namespace {

thread_local std::string g_create_error;

bool is_pow2_kernel_size(int n)
{
    switch(n)
    {
    case 128: case 256: case 512: case 1024: case 2048: case 4096: case 8192: case 16384: case 32768: return true;
    default: return false;
    }
}

// Run-time plan of the any-N kernel: factors of M = N/2, twos grouped up to 16, odd primes as they are.
bool make_any_plan(int n, AnyPlan *plan)
{
    if(n < 128 || (n & 15))
        return false;
    int m = n / 2;
    plan->M = m;
    plan->n_pass = 0;
    int twos = 0;
    while((m & 1) == 0)
    {
        m >>= 1;
        ++twos;
    }
    while(twos > 0)
    {
        const int g = (twos >= 4) ? 4 : twos;
        plan->radix[plan->n_pass++] = 1 << g;
        twos -= g;
    }
    for(int f = 3; m > 1; f += 2)
        while(m % f == 0)
        {
            if(plan->n_pass >= 20)
                return false;
            plan->radix[plan->n_pass++] = f;
            m /= f;
        }
    return true;
}

// Power-of-two sizes 128..32768 take the templated kernels; other multiples of 16 take the any-N kernel as long as
// two N/2-point complex buffers fit in shared memory.
bool supported_fft_size(int n)
{
    if(is_pow2_kernel_size(n))
        return true;
    AnyPlan pl;
    if(!make_any_plan(n, &pl))
        return false;
    return n <= 65536; // sizes whose work buffers exceed shared memory run from a global (L2) scratch
}

// What one call runs: the kernel family, its template arguments and the launch shape the host picks for it.  The rest of the
// shape follows from the template arguments (plan_launch).
enum class Family { fast, team, parity, warp2, v3, wide, fused, anyn };
struct Route {
    Family family;
    int x = 0;                      // EXTRA: options in use (0 / 1); the CTA-per-tick kernel: 0, 1 (out_peak only) or 3
    bool tsm = false, gate = false; // fast: temporal smoothing, silence gate
    int w = 0;                      // fast, warp2: warps per CTA; team: warps per stream
    int r = 1;                      // v3, wide: CTAs per cluster
    int grid = 0;                   // fast, team, warp2, any-N: CTAs
    size_t smem = 0;                // warp2, any-N: dynamic shared memory bytes
    bool scratch = false;           // any-N: work buffers in an L2 scratch instead of shared memory
    bool display = false;           // warp2: the display variant
    bool s16 = false;               // int16 samples (every family: the Pcm<int16_t> instantiation, wf_pcm.cuh)
    int disp_tab_bytes = 0, disp_bytes = 0; // warp2 with display outputs: per-CTA tables, per-warp rows
};

// What routing needs to know about one call, worked out once from its KParams.
struct CallFacts {
    bool display;   // curve points, pixels or minimum requested
    bool opts;      // slope, roll-off, volume, fast peaks, skip mask, peak output or per-tick gravity in use
    int v3_x;       // the CTA-per-tick kernel's level of options: 0, 1 (peak output only) or 3
    bool aligned16; // frames can be loaded in 16-byte units (pcm, stream stride and hop)
    bool db16;      // out_db is 16-byte aligned (the N=2048 kernels write each dB row with one bulk copy)
    bool s16;       // int16 samples
};

// Frames start at 16-byte boundaries (TMA) when pcm does and the stream stride and hop are whole multiples of 16 bytes:
// 4 float samples, 8 int16 samples.  `aligned8` of KParams is the same fact at 8 bytes (launch_range).
CallFacts call_facts(const KParams &kp, bool s16)
{
    const bool opts_but_peak = kp.slope || kp.rolloff || kp.normalize || kp.fast_peaks || kp.skip_mask || kp.g_tab;
    const long long q = s16 ? 7 : 3; // samples per 16 bytes, minus one
    return {.display = kp.out_points || kp.out_pixels || kp.out_min,
            .opts = opts_but_peak || kp.out_peak,
            .v3_x = opts_but_peak ? 3 : (kp.out_peak ? 1 : 0),
            .aligned16 = (((uintptr_t)kp.pcm & 15u) == 0) && ((kp.stream_stride & q) == 0) && ((kp.hop & q) == 0),
            .db16 = ((uintptr_t)kp.out_db & 15u) == 0,
            .s16 = s16};
}

// The display stage's settings (src/source.cpp:1381-1424, 1473-1565) in KParams: set here for the spectrum kernels and for
// wf_render alike, so that both render the same way.  kp.dch must be set; the output pointers are the caller's.
void set_display_params(const wf_engine *e, KParams &kp)
{
    const Tables &t = e->tab;
    kp.interp_idx = e->d_interp_idx;
    kp.interp_w = e->d_interp_w;
    kp.band_widths = e->d_band_widths;
    kp.band_offsets = e->d_band_offsets;
    kp.n_points = t.num_points;
    kp.n_sample = (t.cfg.display_mode == WF_DISPLAY_BAR && t.cfg.interp_mode != WF_INTERP_POINT) ? (int)t.interp_indices.size() : 0;
    kp.scratch_q = t.num_points + (kp.dch * kp.n_sample + 3) / 4;
    kp.taps = t.interp_taps;
    kp.radius = t.interp_radius;
    kp.display_bar = (t.cfg.display_mode == WF_DISPLAY_BAR);
    kp.interp_mode = t.cfg.interp_mode;
    kp.gauss_w = e->d_gauss;
    kp.gauss_radius = t.gauss_radius;
    kp.gauss_size = (int)t.gauss.size();
    kp.gauss_sum = t.gauss_sum;
    kp.filter = (t.cfg.filter_mode == WF_FILTER_GAUSS);
    kp.px_lo = t.px_lo;
    kp.px_hi = t.px_hi;
    kp.px_cpos = t.px_cpos;
    kp.ceiling_f = (float)t.cfg.ceiling_db;
    kp.dbrange_f = (float)(t.cfg.ceiling_db - t.cfg.floor_db);
    kp.mirror = t.cfg.mirror_freq_axis;
}

// Shared memory of the display stage in the fused and any-N kernels: [groups][2][dch <= 2][num_points] floats
size_t display_smem(const KParams &kp, const CallFacts &f, int groups)
{
    return f.display ? (size_t)groups * 4 * (size_t)kp.scratch_q * sizeof(float) : 0;
}

// Cluster size of the wide kernel (wf_wide.cuh) for this launch, 1 = use the one-group-per-stream kernel.
// The wide kernel pays off when there are too few streams to fill the GPU: R CTAs per stream work on R ticks at once.
int pick_wide_r(const wf_engine *e, const KParams &kp, const CallFacts &f)
{
    const KernelRef k = wide_kernel(e->tab.N, e->tab.cfg.capture_channels, 2, f.s16, kp, f.display);
    if(!k.kernel || e->knobs.wide_r == 1 || k.smem > 227 * 1024)
        return 1;
    if(e->knobs.wide_r == 2 || e->knobs.wide_r == 4 || e->knobs.wide_r == 8)
        return e->knobs.wide_r;
    int r = 1;
    while(r < 8 && (long long)kp.n_streams * r < 2LL * e->sm_count && 2 * r <= kp.n_frames)
        r *= 2;
    return r;
}

// Cluster size for the CTA-per-tick kernel (wf_v3.cuh): 1 when the streams alone fill the GPU, else up to 8 CTAs
// (= 8 ticks in flight) per stream.
int pick_v3_r(const wf_engine *e, const KParams &kp)
{
    const int rmin = v3_min_cluster(e->tab.N), wide_r = e->knobs.wide_r;
    if(wide_r == 1 || wide_r == 2 || wide_r == 4 || wide_r == 8)
        return std::max(rmin, wide_r);
    int r = rmin;
    while(r < 8 && (long long)kp.n_streams * r * 3 < 5LL * e->sm_count && 2 * r <= kp.n_frames) // per-tick overhead grows with R
        r *= 2;
    return r;
}

// One CTA per SM; the kernel deals streams round-robin to CTAs first, so each SM gets n_streams/grid (+-1) whole
// streams (the unit of work: EMA state stays on-chip across a stream's frames) and runs min(max_wpc, that) warps.
void fast2048_geometry(int n_streams, int sm_count, int max_wpc, int *warps_per_cta, int *grid)
{
    *grid = std::min(n_streams, sm_count);
    const int per_cta = (n_streams + *grid - 1) / *grid;
    // at least 8 warps even for one stream: the CTA prologue (tables -> shared memory) is spread over the CTA's threads, and
    // with a single warp it dominated the latency of a live tick (1 stream x 1 frame: 19.7 -> ~8 us of kernel time)
    *warps_per_cta = std::max(std::min(8, max_wpc), std::min(max_wpc, per_cta));
}

// Warps per stream of the N=2048 team kernel (wf_team2048.cuh), 1 = the warp-per-stream kernel.  Fewer streams than SMs x 16
// warps: a team of W warps per stream works on W ticks at once.  Up to 8 streams per SM: 16 / W = 1, 2 or 4 teams per SM (a
// team takes its streams one after the other); measured (profiles/r02_layouts.txt) 256 x 256: 142 -> 272 M spectra/s,
// 512 x 128: 200 -> 310 M, 1024 x 64: 289 -> 332 M.
int pick_team_w(const wf_engine *e, const KParams &kp)
{
    const int team_w = e->knobs.team_w;
    if(team_w == 1)
        return 1;
    int W = 1;
    const int per_sm = (kp.n_streams + e->sm_count - 1) / e->sm_count;
    if(per_sm <= 8)
        W = (per_sm <= 1) ? 16 : (per_sm == 2) ? 8 : 4;
    if(team_w == 4 || team_w == 8 || team_w == 16)
        W = team_w;
    while(W > 1 && W > kp.n_frames)
        W /= 2;
    return (W == 2) ? 1 : W;
}

// Warps per CTA of the warp-per-stream kernel for N = 2*L*P (wf_warp2.cuh) and its shared memory, into `r`; false when not
// even one warp's display rows fit (the call then goes to the next family).
bool fit_warp2(const wf_engine *e, const KParams &kp, bool display, Route &r)
{
    constexpr size_t kMaxSmem = 227 * 1024; // opt-in shared memory per CTA on sm_90
    fast2048_geometry(kp.n_streams, e->sm_count, 16, &r.w, &r.grid);
    if(display)
    {
        // shared memory of the display variant (layout in wf_warp2.cuh): per CTA the setup tables, per warp the tick's dB
        // row, the bar sample points and — only for the Gaussian / pixel / minimum outputs — two rows of points + scratch
        const size_t tab = display_table_floats(kp);
        const bool need_pts = kp.filter || kp.out_pixels || kp.out_min;
        const size_t per_warp = (size_t)e->tab.B + (size_t)kp.n_sample + (need_pts ? 2 * (size_t)kp.n_points + 64 : 0);
        r.disp_tab_bytes = (int)((tab * sizeof(float) + 127) / 128 * 128);
        r.disp_bytes = (int)((per_warp * sizeof(float) + 127) / 128 * 128);
    }
    // the display rows cost warps per SM at the largest sizes; the streams simply take more rounds
    while(r.w > 1 && e->warp2.smem_bytes(r.w, r.disp_tab_bytes, r.disp_bytes) > kMaxSmem)
        --r.w;
    r.smem = e->warp2.smem_bytes(r.w, r.disp_tab_bytes, r.disp_bytes);
    return r.smem <= kMaxSmem;
}

// The kernel a call runs, in order of precedence: the N=2048 team and warp-per-stream kernels, the N=16384 parity
// clusters, the warp-per-stream kernel of the other sizes (and of display outputs), the CTA-per-tick clusters, the wide
// clusters, the fused kernel of the power-of-two sizes and the any-N kernel.
Route choose_route(const wf_engine *e, const KParams &kp, const CallFacts &f)
{
    const Tables &t = e->tab;
    const SpectrumKnobs &k = e->knobs;
    const int N = t.N, cc = t.cfg.capture_channels;
    const bool mono = (cc == 1) && !t.cfg.stereo, x = f.opts;
    if(N == 2048 && mono && kp.out_db && !f.display && f.aligned16 && f.db16 && !k.force_generic)
    {
        if(const int W = pick_team_w(e, kp); W > 1)
            return {.family = Family::team, .x = x, .w = W, .grid = std::min(e->sm_count, kp.n_streams)};
        Route r{.family = Family::fast, .x = x, .tsm = kp.tsmooth != 0, .gate = kp.gate != 0};
        fast2048_geometry(kp.n_streams, e->sm_count, fast::kMaxWarpsPerCta, &r.w, &r.grid);
        return r;
    }
    // N = 16384 (config 5): a cluster of two CTAs per stream splits the bins by parity, each on the spill-free N=8192 plan
    if(N == 16384 && k.par16384 && k.v3 && e->d_tw0 && mono && kp.out_db && !f.display && !k.force_generic)
        return {.family = Family::parity, .x = x};
    // Non-power-of-two sizes with a compiled two-pass plan (wf_warp2.cuh): same launch shape as the N=2048 kernel.  With
    // display outputs (curve points / bars / pixels / minimum) the same kernel runs the render-time stages per warp; that
    // variant also takes the power-of-two sizes 512 / 1024 / 2048 (config 1: N=1024, 26 bars).
    const bool pow2 = is_pow2_kernel_size(N);
    if(k.warp2 && mono && f.aligned16 && e->warp2.L &&
       (f.display ? (k.warp2_display && !k.force_generic) : (!pow2 && kp.out_db)))
    {
        Route r{.family = Family::warp2, .x = x, .display = f.display};
        if(fit_warp2(e, kp, f.display, r))
            return r;
    }
    if(k.v3 && e->d_tw1 != nullptr && v3_kernel(N, cc, 8, f.v3_x, f.s16, kp, f.display).smem <= 227 * 1024)
        return {.family = Family::v3, .x = f.v3_x, .r = pick_v3_r(e, kp)};
    if(const int R = pick_wide_r(e, kp, f); R > 1)
        return {.family = Family::wide, .r = R};
    if(pow2)
        return {.family = Family::fused};
    // any other multiple of 16: the run-time mixed-radix kernel, its work buffers in shared memory or in an L2 scratch
    const size_t extra = display_smem(kp, f, 1), work = (size_t)e->any.M * 16;
    const bool in_smem = work + extra <= 200 * 1024;
    return {.family = Family::anyn, .grid = std::min(kp.n_streams, e->sm_count * (in_smem ? 8 : 2)),
            .smem = in_smem ? work + extra : extra, .scratch = !in_smem};
}

// How a route launches: the kernel instantiation, its shape and launch mode, the argument it takes after KParams, and its
// name (wf_last_kernel_name).
struct Launch {
    enum class Arg { none, tw3, any }; // after KParams: nothing, the v3 twiddles (v3::Tw3) or the any-N plan (AnyPlan)
    const void *kernel = nullptr;
    unsigned grid = 0, block = 0;
    size_t smem = 0;
    LaunchMode mode{};
    Arg arg = Arg::none;
    std::string name;
};

// The launch of route r for this call.  The instantiation, the shape and the name all come from the same fields of r, so the
// name describes the kernel that runs.
Launch plan_launch(const wf_engine *e, const Route &r, const KParams &kp, const CallFacts &f)
{
    using Arg = Launch::Arg;
    const int N = e->tab.N, cc = e->tab.cfg.capture_channels;
    const unsigned S = (unsigned)kp.n_streams;
    Launch l;
    KernelRef k;
    char buf[128];
    switch(r.family)
    {
    case Family::fast:
        k = fast2048_kernel(r.tsm, r.gate, r.x, r.s16);
        l = {k.kernel, (unsigned)r.grid, r.w * 32u, (size_t)fast::smem_bytes(r.w), {.pdl = true}};
        snprintf(buf, sizeof buf, "stft2048_fast_kernel<%d,%d,%d,%d> grid %d x %d warps", fast::kMaxWarpsPerCta, (int)r.tsm,
                 (int)r.gate, r.x, r.grid, r.w);
        break;
    case Family::team:
        k = team2048_kernel(r.w, r.x, r.s16);
        l = {k.kernel, (unsigned)r.grid, k.block, k.smem, {.pdl = true}};
        snprintf(buf, sizeof buf, "stft2048_team_kernel<%d,%d> grid %d x %d teams", r.w, r.x, r.grid, 16 / r.w);
        break;
    case Family::parity:
        k = par16384_kernel(r.x, r.s16);
        l = {k.kernel, 2 * S, k.block, k.smem, {}, Arg::tw3};
        snprintf(buf, sizeof buf, "stft16384_parity_kernel<%d> %d clusters of 2", r.x, kp.n_streams);
        break;
    case Family::warp2:
        l = {e->warp2.kernel[r.s16][r.x][r.display], (unsigned)r.grid, r.w * 32u, r.smem, {.pdl = true}};
        snprintf(buf, sizeof buf, "stft_warp2_kernel<%d,%d%s> N=%d grid %d x %d warps", e->warp2.L, e->warp2.P,
                 r.display ? ",display" : "", N, r.grid, r.w);
        break;
    case Family::v3:
        k = v3_kernel(N, cc, r.r, r.x, r.s16, kp, f.display);
        l = {k.kernel, S * r.r, k.block, k.smem, {.cluster = (unsigned)r.r}, Arg::tw3};
        snprintf(buf, sizeof buf, "stft_v3_kernel<%d,%d,%d,%d>", N, cc, r.r, r.x);
        break;
    case Family::wide:
        k = wide_kernel(N, cc, r.r, r.s16, kp, f.display);
        l = {k.kernel, S * r.r, k.block, k.smem, {.cluster = (unsigned)r.r}};
        snprintf(buf, sizeof buf, "stft_wide_kernel<%d,%d,%d>", N, cc, r.r);
        break;
    case Family::fused:
    {
        int groups = 1;
        k = fused_kernel(N, cc, r.s16, &groups);
        l = {k.kernel, (S + groups - 1) / groups, k.block, k.smem + display_smem(kp, f, groups)};
        snprintf(buf, sizeof buf, "stft_fused_kernel<%d,%d>", N, cc);
        break;
    }
    case Family::anyn:
        k = anyn_kernel(cc, r.s16);
        l = {k.kernel, (unsigned)r.grid, k.block, r.smem, {}, Arg::any};
        snprintf(buf, sizeof buf, "stft_anyn_kernel<%d> N=%d", cc, N);
        break;
    }
    l.name = r.s16 ? std::string(buf) + " s16" : std::string(buf);
    return l;
}

// Write out every implicit m_decibels mirror (see materialize_hold_kernel) before something other than the N=2048
// warp-per-stream kernel looks at hold_db.
int materialize_hold(wf_engine *e, cudaStream_t st)
{
    if(!e->hold_implicit)
        return WF_OK;
    const Tables &t = e->tab;
    const int S = t.cfg.max_streams;
    WF_CHECK(e, launch_kernel(materialize_hold_kernel, e->device, std::min(S, e->sm_count * 8), 256, 0, st, {}, e->d_state,
                              e->d_hold, e->d_flags, S, t.B, t.output_channels, t.db_min));
    e->launches++;
    e->hold_implicit = e->hold_replayed;
    return WF_OK;
}

// Fresh streams (wf_create): m_tsmooth_buf = 0, m_decibels = DB_MIN, m_last_silent = false (src/source.cpp:1176-1180, 1236).
int init_state(wf_engine *e, int first, int count, cudaStream_t st)
{
    const Tables &t = e->tab;
    const int cc = t.cfg.capture_channels, och = t.output_channels, B = t.B;
    WF_CHECK(e, cudaMemsetAsync(e->d_state + (size_t)first * cc * B, 0, (size_t)count * cc * B * sizeof(float), st));
    int rc = fill_device(e, e->d_hold + (size_t)first * och * B, (long long)count * och * B, t.db_min, st);
    if(rc)
        return rc;
    // flags: bit0 last_silent; bit1/2: previous outputs all <= floor-10 (DB_MIN is)
    const bool below = !(t.db_min > (float)(t.cfg.floor_db - 10));
    WF_CHECK(e, cudaMemsetAsync(e->d_flags + first, below ? 6 : 0, (size_t)count, st));
    return WF_OK;
}

// A ring call's window (wf_splice.hpp) with ring length R = N + D: C[hop .. hop + (T-1)*hop + N), the call's frames in the
// plain layout, reaching at least to R so that it holds the part of the next ring that predates the call (D > T*hop).  Its
// length is 0 when hop >= R: every frame then lies wholly in the new samples and the kernel reads them in place.
long long ring_window_len(int N, int D, int hop, int T)
{
    const long long R = (long long)N + D;
    if(hop >= R)
        return 0;
    return std::max((long long)(T - 1) * hop + N, R - hop);
}

// The capture rings, allocated and zeroed (the plugin's start-up zeros, src/source.cpp:1243-1248) on first use.  A first use
// that is being captured zeroes them at once on the engine's own stream, outside the graph, which must not zero them again
// on every replay.
int ensure_ring(wf_engine *e, cudaStream_t st)
{
    if(e->d_ring.p)
        return WF_OK;
    const Tables &t = e->tab;
    const size_t n = (size_t)t.cfg.max_streams * t.cfg.capture_channels * (t.N + e->D);
    if(int rc = e->d_ring.reserve(e, n))
        return rc;
    if(!e->capturing)
    {
        WF_CHECK(e, cudaMemsetAsync(e->d_ring, 0, n * sizeof(float), st));
        return WF_OK;
    }
    WF_CHECK(e, outside_capture(e, [&] {
        const cudaError_t err = cudaMemsetAsync(e->d_ring, 0, n * sizeof(float), e->stream);
        return err ? err : cudaStreamSynchronize(e->stream);
    }));
    return WF_OK;
}

// wf_get_ring / wf_set_ring: checks, the rings, and the stream order of the copies
int ring_access(wf_engine *e, int32_t first, int32_t count, const void *samples)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    if(int rc = check_slot_range(e, first, count, e->tab.cfg.max_streams, "ring"))
        return rc;
    if(count > 0 && !samples)
        return fail(e, WF_ERR_INVALID_ARG, "samples is null");
    WF_CHECK(e, cudaSetDevice(e->device));
    if(int rc = ensure_ring(e, e->stream))
        return rc;
    WF_CHECK(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

// wf_get_state (set = false) / wf_set_state (set = true): one copy and one launch, not counted as one of the engine's
int spectrum_state(wf_engine *e, int32_t first, int32_t count, const float *tsmooth, const float *hold_db,
                   const uint8_t *flags, bool set)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    const Tables &t = e->tab;
    if(int rc = check_slot_range(e, first, count, t.cfg.max_streams, "state"))
        return rc;
    WF_CHECK(e, cudaSetDevice(e->device));
    if(int rc = materialize_hold(e, e->stream))
        return rc;
    WF_CHECK(e, cudaStreamSynchronize(e->stream));
    const size_t n = (size_t)count, cc = (size_t)t.cfg.capture_channels, och = (size_t)t.output_channels, B = (size_t)t.B;
    StateSections io;
    const int i_tsmooth = io.add(tsmooth, n * cc * B * sizeof(float));
    const int i_hold = io.add(hold_db, n * och * B * sizeof(float));
    const int i_flags = io.add(flags, n);
    if(io.empty())
        return WF_OK;
    if(int rc = io.reserve(e, e->s_state, e->h_state))
        return rc;
    // the legacy default stream orders the state call after the work callers enqueued on blocking streams (torch's default)
    return io.run(e, cudaStreamLegacy, set, [&] {
        return launch_kernel(set ? spectrum_state_kernel<true> : spectrum_state_kernel<false>, e->device,
                             std::min(count, e->sm_count * 8), 256, 0, cudaStreamLegacy, {}, e->d_state + first * cc * B,
                             e->d_hold + first * och * B, e->d_flags + first, io.dev<float>(i_tsmooth),
                             io.dev<float>(i_hold), io.dev<unsigned char>(i_flags), count, (int)cc, (int)och,
                             t.display_channels, (int)B, (float)(t.cfg.floor_db - 10));
    });
}

} // namespace

extern "C" {

int wf_abi_version(void) { return WF_ABI_VERSION; }

const char *wf_strerror(int status)
{
    switch(status)
    {
    case WF_OK: return "ok";
    case WF_ERR_INVALID_ARG: return "invalid argument";
    case WF_ERR_UNSUPPORTED_FFT_SIZE: return "unsupported fft_size (supported: multiples of 16 from 128 to 65536)";
    case WF_ERR_CUDA: return "CUDA error";
    case WF_ERR_NO_DEVICE: return "no CUDA device (this engine has no CPU fallback)";
    case WF_ERR_OOM: return "out of device memory";
    case WF_ERR_CAPACITY: return "stream range exceeds max_streams";
    case WF_ERR_ABI: return "struct_size mismatch (ABI)";
    default: return "unknown status";
    }
}

const char *wf_last_error(const wf_engine *e) { return e ? e->last_error.c_str() : g_create_error.c_str(); }

void wf_config_init(wf_config *c)
{
    // plugin defaults, src/source.cpp:119-174
    memset(c, 0, sizeof(*c));
    c->struct_size = (uint32_t)sizeof(wf_config);
    c->device = -1;
    c->max_streams = 1;
    c->sample_rate = 48000;
    c->capture_channels = 2;
    c->fft_size = 4096;
    c->window = WF_WINDOW_HANN;
    c->sine_exponent = 2;
    c->tsmoothing = WF_TSMOOTH_EXPONENTIAL;
    c->gravity = 0.65f;
    c->fast_peaks = 0;
    c->slope = 0.0f;
    c->rolloff_q = 0.0f;
    c->rolloff_rate = 0.0f;
    c->cutoff_low = 30;
    c->cutoff_high = 17500;
    c->floor_db = -65;
    c->ceiling_db = 0;
    c->stereo = 0;
    c->normalize_volume = 0;
    c->volume_target = -8.0f;
    c->max_gain = 30.0f;
    c->silence_gate = 1;
    c->display_mode = WF_DISPLAY_CURVE;
    c->width = 800;
    c->bar_width = 24;
    c->bar_gap = 6;
    c->log_scale = 1;
    c->mirror_freq_axis = 0;
    c->interp_mode = WF_INTERP_CATROM;
    c->filter_mode = WF_FILTER_NONE;
    c->filter_radius = 1.5f;
    c->height = 225;
    c->channel_spacing = 0;
    c->rounded_caps = 0;
    c->min_bar_height = 0;
    c->sync_offset_ms = 0;
}

int wf_create(const wf_config *cfg, wf_engine **out)
{
    if(!cfg || !out)
        return WF_ERR_INVALID_ARG;
    *out = nullptr;
    // the current struct or the previous one, which ends before sync_offset_ms (no offset)
    wf_config cv;
    if(!accept_struct(cfg, {offsetof(wf_config, sync_offset_ms)}, cv))
        return WF_ERR_ABI;
    return create_engine(out, g_create_error, wf_destroy, [&](wf_engine *e) -> int {
        if(!sync_offset_ok(cv.sync_offset_ms))
            return fail(e, WF_ERR_INVALID_ARG, "sync_offset_ms %d outside [-1000, 1000]", cv.sync_offset_ms);
        const char *why = nullptr;
        int rc = build_tables(cv, e->tab, &why);
        if(rc != WF_OK)
            return fail(e, rc, "%s", why ? why : "bad config");
        if(!supported_fft_size(e->tab.N))
            return fail(e, WF_ERR_UNSUPPORTED_FFT_SIZE, "fft_size %d unsupported", e->tab.N);
        if((rc = open_device(e, cv.device)))
            return rc;
        e->D = sync_delay(e->tab.cfg.sample_rate, cv.sync_offset_ms);
        e->owed.assign((size_t)e->tab.cfg.max_streams, e->D);
        if(e->D > 0 && (rc = e->d_owed.upload(e, e->owed)))
            return rc;
        e->warp2 = warp2_plan(e->tab.N);
        if(!is_pow2_kernel_size(e->tab.N))
            make_any_plan(e->tab.N, &e->any);

        const Tables &t = e->tab;
        std::vector<float> tw1, tw2, tw0; // stay empty (and d_tw1 null) for sizes without the CTA-per-tick kernel
        v3_build_twiddles(t.N, tw1, tw2, tw0);
        for(auto [buf, v] : {std::pair{&e->d_window, &t.window}, {&e->d_slope, &t.slope}, {&e->d_rolloff, &t.rolloff},
                             {&e->d_tw, &t.tw}, {&e->d_tw_post, &t.tw_post}, {&e->d_tw1, &tw1}, {&e->d_tw2, &tw2},
                             {&e->d_tw0, &tw0}, {&e->d_interp_idx, &t.interp_indices}, {&e->d_interp_w, &t.interp_weights},
                             {&e->d_gauss, &t.gauss}})
            if((rc = buf->upload(e, *v)))
                return rc;
        for(auto [buf, v] : {std::pair{&e->d_band_widths, &t.band_widths}, {&e->d_band_offsets, &t.band_offsets}})
            if((rc = buf->upload(e, *v)))
                return rc;

        const size_t S = (size_t)t.cfg.max_streams;
        if((rc = e->d_state.reserve(e, S * t.cfg.capture_channels * t.B)))
            return rc;
        if((rc = e->d_hold.reserve(e, S * t.output_channels * t.B)))
            return rc;
        if((rc = e->d_flags.reserve(e, S)))
            return rc;
        if((rc = init_state(e, 0, (int)S, e->stream)))
            return rc;
        WF_CHECK(e, cudaStreamSynchronize(e->stream));
        return WF_OK;
    });
}

void wf_destroy(wf_engine *e)
{
    if(!e)
        return;
    if(e->stream)
    {
        cudaSetDevice(e->device);
        cudaStreamSynchronize(e->stream);
    }
    for(auto ev : e->chunk_in)
        if(ev)
            cudaEventDestroy(ev);
    for(auto ev : e->chunk_k)
        if(ev)
            cudaEventDestroy(ev);
    if(e->ev_fork)
        cudaEventDestroy(e->ev_fork);
    if(e->ev_join)
        cudaEventDestroy(e->ev_join);
    if(e->s_h2d)
        cudaStreamDestroy(e->s_h2d);
    if(e->s_d2h)
        cudaStreamDestroy(e->s_d2h);
    delete e;
}

static int64_t copy_table(const Tables &t, int which, float *out, int64_t capacity);
static void fill_info(const Tables &t, wf_info *info, int device, int sm_count);

int wf_get_info(const wf_engine *e, wf_info *info)
{
    if(!e || !info)
        return WF_ERR_INVALID_ARG;
    fill_info(e->tab, info, e->device, e->sm_count);
    return WF_OK;
}

int64_t wf_get_table(const wf_engine *e, int which, float *out, int64_t capacity)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    return copy_table(e->tab, which, out, capacity);
}

float wf_gravity(const wf_engine *e, float seconds) { return e ? gravity_for(e->tab.cfg, seconds) : 0.0f; }

static int64_t copy_table(const Tables &t, int which, float *out, int64_t capacity)
{
    const void *src = nullptr;
    int64_t n = 0;
    switch(which)
    {
    case WF_TABLE_WINDOW: src = t.window.data(); n = (int64_t)t.window.size(); break;
    case WF_TABLE_SLOPE: src = t.slope.data(); n = (int64_t)t.slope.size(); break;
    case WF_TABLE_ROLLOFF: src = t.rolloff.data(); n = (int64_t)t.rolloff.size(); break;
    case WF_TABLE_INTERP_INDICES: src = t.interp_indices.data(); n = (int64_t)t.interp_indices.size(); break;
    case WF_TABLE_INTERP_WEIGHTS: src = t.interp_weights.data(); n = (int64_t)t.interp_weights.size(); break;
    case WF_TABLE_BAND_WIDTHS: src = t.band_widths.data(); n = (int64_t)t.band_widths.size(); break;
    case WF_TABLE_GAUSS: src = t.gauss.data(); n = (int64_t)t.gauss.size(); break;
    default: return WF_ERR_INVALID_ARG;
    }
    if(out && n > 0)
    {
        if(capacity < n)
            return WF_ERR_INVALID_ARG;
        memcpy(out, src, (size_t)n * 4);
    }
    return n;
}

static void fill_info(const Tables &t, wf_info *info, int device, int sm_count)
{
    info->fft_size = t.N;
    info->bins = t.B;
    info->capture_channels = t.cfg.capture_channels;
    info->output_channels = t.output_channels;
    info->display_channels = t.display_channels;
    info->num_points = t.num_points;
    info->num_bars = t.num_bars;
    info->interp_taps = t.interp_taps;
    info->n_interp_indices = (int32_t)t.interp_indices.size();
    info->window_sum = t.window_sum;
    info->db_min = t.db_min;
    info->device = device;
    info->sm_count = sm_count;
}

int64_t wf_preview_table(const wf_config *cfg, int which, float *out, int64_t capacity, wf_info *info)
{
    if(!cfg)
        return WF_ERR_INVALID_ARG;
    wf_config cv;
    if(!accept_struct(cfg, {offsetof(wf_config, sync_offset_ms)}, cv))
        return WF_ERR_ABI;
    if(!sync_offset_ok(cv.sync_offset_ms))
    {
        g_create_error = "sync_offset_ms outside [-1000, 1000]";
        return WF_ERR_INVALID_ARG;
    }
    Tables t;
    const char *why = nullptr;
    int rc = build_tables(cv, t, &why);
    if(rc != WF_OK)
    {
        g_create_error = why ? why : "bad config";
        return rc;
    }
    if(info)
        fill_info(t, info, -1, -1);
    return copy_table(t, which, out, capacity);
}

// Runs a route: writes out the implicit m_decibels mirrors first unless the route is one of the N=2048 kernels (the other
// kernels read hold_db as it is), sets the route's own KParams fields, launches, and names the kernel.  A captured call of
// another route on an N=2048 engine always includes that pass: the graph may be replayed after an N=2048 kernel left
// mirrors implicit, whatever the host knows now (the pass only touches streams that carry flags bit 3).
static int launch_route(wf_engine *e, const Route &r, const Launch &l, KParams kp, cudaStream_t st)
{
    if(r.family != Family::fast && r.family != Family::team)
    {
        e->hold_implicit = e->hold_implicit || (e->capturing && e->tab.N == 2048);
        if(int rc = materialize_hold(e, st))
            return rc;
    }
    AnyPlan plan = e->any;
    plan.scratch = nullptr;
    switch(r.family)
    {
    case Family::fast:
    case Family::team:
        kp.split = e->knobs.split ? 1 : 0;
        kp.lazy_hold = 1;
        e->hold_implicit = true;
        e->hold_replayed = e->hold_replayed || e->capturing;
        break;
    case Family::warp2:
        kp.split = e->knobs.split ? 1 : 0;
        kp.disp_tab_bytes = r.disp_tab_bytes;
        kp.disp_bytes = r.disp_bytes;
        break;
    case Family::anyn:
        if(r.scratch)
        {
            if(int rc = e->s_scratch.reserve(e, (size_t)r.grid * 2 * plan.M * 2))
                return rc;
            plan.scratch = reinterpret_cast<float2 *>(e->s_scratch.p);
        }
        break;
    default: break;
    }
    v3::Tw3 tw{reinterpret_cast<const float2 *>(e->d_tw1.p), reinterpret_cast<const float2 *>(e->d_tw2.p),
               reinterpret_cast<const float2 *>(e->d_tw0.p)};
    void *args[2] = {&kp, nullptr};
    if(l.arg == Launch::Arg::tw3)
        args[1] = &tw;
    else if(l.arg == Launch::Arg::any)
        args[1] = &plan;
    WF_CHECK(e, launch_kernel(l.kernel, e->device, l.grid, l.block, l.smem, st, l.mode, args));
    e->launches++;
    e->last_kernel = l.name;
    return WF_OK;
}

// pcm + `samples` samples of the batch's format (the pointer stays `const float *`, as in wf_batch and KParams)
static const float *pcm_offset(const float *pcm, long long samples, bool s16)
{
    return reinterpret_cast<const float *>(reinterpret_cast<const char *>(pcm) + samples * (s16 ? 2 : 4));
}

// `buf` grown to at least `bytes` bytes (the staging buffers count floats)
static int reserve_bytes(wf_engine *e, DevBuf<float> &buf, size_t bytes)
{
    return buf.reserve(e, (bytes + sizeof(float) - 1) / sizeof(float));
}

// One buffer of a wf_batch other than pcm: its pointer field, which way a staged call copies it, its extent and the engine's
// staging buffer for it.  PCM is strided rather than contiguous per stream, so it keeps its own span (wf_process_async) and
// offset (launch_range).
struct BatchBuf {
    size_t field;         // offsetof(wf_batch, <pointer>)
    bool in;              // read by the kernels (host -> device) or written by them (device -> host)
    bool per_stream;      // `bytes` per stream of the call, or for the whole call (out_peak)
    size_t bytes;
    DevBuf<float> *stage;

    // the batch's pointer in this field, as bytes (every data pointer of wf_batch has the same representation)
    char *of(const wf_batch &b) const
    {
        char *p;
        memcpy(&p, reinterpret_cast<const char *>(&b) + field, sizeof p);
        return p;
    }
    void set(wf_batch &b, const void *p) const { memcpy(reinterpret_cast<char *>(&b) + field, &p, sizeof p); }
};
using BatchBufs = std::array<BatchBuf, wf_engine::kBatchBufs>;

// The buffers of a call of n_frames = T, in wf_batch's order; the host path reserves, copies and offsets them from this
// table alone.
static BatchBufs batch_bufs(wf_engine *e, size_t T)
{
    const Tables &t = e->tab;
    const size_t f = sizeof(float), rows = T * t.display_channels;
    return {{{offsetof(wf_batch, input_rms), true, true, T * f, &e->s_rms},
             {offsetof(wf_batch, skip_mask), true, true, T, &e->s_skip},
             {offsetof(wf_batch, out_db), false, true, rows * t.B * f, &e->s_out_db},
             {offsetof(wf_batch, out_points), false, true, rows * t.num_points * f, &e->s_out_points},
             {offsetof(wf_batch, out_silent), false, true, T, &e->s_silent},
             {offsetof(wf_batch, out_peak), false, false, T * f, &e->s_peak},
             {offsetof(wf_batch, out_pixels), false, true, rows * t.num_points * f, &e->s_px},
             {offsetof(wf_batch, out_min), false, true, T * 2 * f, &e->s_min}}};
}

// Runs streams [s0, s0+count) of `b`, whose pointers the device can address: the caller's own, or the staging buffers of a
// host batch laid out as the caller's buffers.  Every pointer is offset to stream s0 here.
static int launch_range(wf_engine *e, const wf_batch *b, const BatchBufs &bufs, cudaStream_t st, int s0, int count,
                        const float *g_tab_dev)
{
    const Tables &t = e->tab;
    const int cc = t.cfg.capture_channels, och = t.output_channels, B = t.B;
    const bool s16 = b->pcm_format == WF_PCM_S16, ring = b->capture_ring == WF_CAPTURE_RING;
    wf_batch at = *b; // b's buffers from stream s0 on
    for(const BatchBuf &u : bufs)
        if(char *p = u.of(*b); p && u.per_stream)
            u.set(at, p + (size_t)s0 * u.bytes);
    const float *new_pcm = pcm_offset(b->pcm, (long long)s0 * b->stream_stride, s16);
    KParams kp{};
    kp.pcm = new_pcm;
    kp.stream_stride = b->stream_stride;
    kp.channel_stride = b->channel_stride;
    // A ring call runs the plain kernel on plain-layout frames: the splice's window (hop < R), or the new samples themselves
    // with frame t at new[t*hop + hop - R] (hop >= R), R = N + D.  The alignment facts below are those of what the kernel reads.
    const int R = t.N + e->D;
    const long long win_len = ring ? ring_window_len(t.N, e->D, b->hop, b->n_frames) : 0;
    const long long win_cs = splice_stride(win_len, s16);
    if(win_cs > 0)
    {
        kp.pcm = pcm_offset(e->s_window, (long long)s0 * cc * win_cs, s16);
        kp.stream_stride = cc * win_cs;
        kp.channel_stride = win_cs;
    }
    else if(ring)
        kp.pcm = pcm_offset(new_pcm, (long long)b->hop - R, s16);
    kp.n_streams = count;
    kp.n_frames = b->n_frames;
    kp.hop = b->hop;
    // every frame starts at an 8-byte boundary: 2 float samples, 4 int16 samples
    const long long q = s16 ? 3 : 1;
    kp.aligned8 = (((uintptr_t)kp.pcm & 7u) == 0) && ((kp.stream_stride & q) == 0) && ((kp.channel_stride & q) == 0) &&
                  ((b->hop & q) == 0);
    kp.input_rms = at.input_rms;
    kp.skip_mask = at.skip_mask;
    // a ring call during the sync offset's start-up skips through its own mask (the caller's ORed in, the splice writes
    // it), routed as such
    const bool startup = ring && e->startup;
    unsigned char *startup_mask = startup ? e->s_mask + (size_t)s0 * b->n_frames : nullptr;
    if(startup)
        kp.skip_mask = startup_mask;
    kp.window = e->d_window;
    kp.window2 = reinterpret_cast<const float2 *>(e->d_window.p);
    kp.tw = reinterpret_cast<const float2 *>(e->d_tw.p);
    kp.tw_post = reinterpret_cast<const float2 *>(e->d_tw_post.p);
    kp.slope = e->d_slope;
    kp.rolloff = e->d_rolloff;
    const size_t slot = (size_t)b->first_stream + (size_t)s0;
    kp.state = e->d_state + slot * cc * B;
    kp.hold_db = e->d_hold + slot * och * B;
    kp.flags = e->d_flags + slot;
    kp.out_db = at.out_db;
    kp.out_points = at.out_points;
    kp.out_silent = at.out_silent;
    kp.out_peak = at.out_peak;
    kp.out_pixels = at.out_pixels;
    kp.out_min = at.out_min;
    kp.coef_half = (2.0f / t.window_sum) * 0.5f; // mag_coefficient/2: the split pass leaves 2*X (src/source_generic.cpp:110)
    kp.g = (t.cfg.tsmoothing == WF_TSMOOTH_NONE) ? 0.0f : gravity_for(t.cfg, b->seconds);
    kp.g2 = 1.0f - kp.g;
    kp.g_tab = reinterpret_cast<const float2 *>(g_tab_dev);
    kp.tsmooth = t.cfg.tsmoothing != WF_TSMOOTH_NONE;
    kp.fast_peaks = t.cfg.fast_peaks;
    kp.stereo = t.cfg.stereo;
    kp.och = och;
    kp.dch = t.display_channels;
    kp.gate = t.cfg.silence_gate;
    kp.floor_m10 = (float)(t.cfg.floor_db - 10);
    kp.db_min = t.db_min;
    kp.normalize = t.cfg.normalize_volume;
    kp.vol_target = t.cfg.volume_target;
    kp.max_gain = t.cfg.max_gain;
    kp.write_hold = 1;
    set_display_params(e, kp);

    const CallFacts f = call_facts(kp, s16);
    Route r = choose_route(e, kp, f);
    r.s16 = s16;
    const Launch l = plan_launch(e, r, kp, f);
    if(ring)
    {
        Splice sp{};
        sp.hist = e->d_ring + slot * cc * R;
        sp.win = win_cs > 0 ? const_cast<float *>(kp.pcm) : nullptr;
        sp.pcm = new_pcm;
        sp.stream_stride = b->stream_stride;
        sp.channel_stride = b->channel_stride;
        sp.win_cs = win_cs;
        sp.ws = b->hop;
        sp.wl = win_len;
        sp.L = (long long)b->n_frames * b->hop;
        sp.R = R;
        if(startup)
        {
            sp.owed = e->d_owed + slot;
            sp.mask = startup_mask;
            sp.caller = at.skip_mask;
            sp.T = b->n_frames;
            sp.hop = b->hop;
        }
        WF_CHECK(e, launch_splice(sp, e->device, count, cc, s16, st));
        e->launches++;
    }
    if(int rc = launch_route(e, r, l, kp, st))
        return rc;
    if(ring)
        e->last_kernel += " ring";
    return WF_OK;
}



int wf_process_async(wf_engine *e, const wf_batch *b_in, void *cuda_stream)
{
    if(!e || !b_in)
        return WF_ERR_INVALID_ARG;
    NvtxRange nvtx("wf_process");
    // the current struct or the one ending before pcm_format (float PCM).  capture_ring took the previous struct's tail
    // padding, so the previous size is the current one.
    wf_batch bv;
    if(!accept_struct(b_in, {offsetof(wf_batch, pcm_format)}, bv))
        return fail(e, WF_ERR_ABI, "wf_batch.struct_size %u != %zu", b_in->struct_size, sizeof(wf_batch));
    const wf_batch *b = &bv;
    const Tables &t = e->tab;
    const int cc = t.cfg.capture_channels, N = t.N;
    if(b->n_streams < 0 || b->n_frames < 0 || b->hop < 1)
        return fail(e, WF_ERR_INVALID_ARG, "n_streams/n_frames must be >= 0 and hop >= 1");
    if(int rc = check_slot_range(e, b->first_stream, b->n_streams, t.cfg.max_streams, "stream"))
        return rc;
    if(b->n_streams == 0 || b->n_frames == 0)
        return WF_OK;
    if(!b->pcm)
        return fail(e, WF_ERR_INVALID_ARG, "pcm is null");
    if(b->stream_stride < 0 || b->channel_stride < 0)
        return fail(e, WF_ERR_INVALID_ARG, "negative strides are not supported");
    size_t sample_bytes = 0;
    if(int rc = pcm_sample_bytes(e, b->pcm_format, b->pcm, &sample_bytes))
        return rc;
    const bool s16 = b->pcm_format == WF_PCM_S16;
    if(t.cfg.normalize_volume && !b->input_rms)
        return fail(e, WF_ERR_INVALID_ARG, "normalize_volume is set but the batch carries no input_rms (m_input_rms per tick: "
                                              "wf_meter in WF_METER_INPUT_RMS mode, or the host's own update_input_rms)");
    if((b->out_points || b->out_pixels || b->out_min) && t.num_points <= 0)
        return fail(e, WF_ERR_INVALID_ARG, "display outputs requested but the engine has no display points");

    WF_CHECK(e, cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    WF_CHECK(e, begin_call(e, st));
    const size_t S = (size_t)b->n_streams, T = (size_t)b->n_frames;
    const bool ring = b->capture_ring == WF_CAPTURE_RING;
    const BatchBufs bufs = batch_bufs(e, T);
    if(int rc = refuse_pageable(e, {b->pcm, bufs[0].of(*b), bufs[1].of(*b), bufs[2].of(*b), bufs[3].of(*b), bufs[4].of(*b),
                                    bufs[5].of(*b), bufs[6].of(*b), bufs[7].of(*b)}))
        return rc;
    if(ring)
    {
        if(int rc = ensure_ring(e, st))
            return rc;
        // the window of every stream of the call (chunks of a staged call take their own parts of it)
        const size_t win = S * cc * (size_t)splice_stride(ring_window_len(N, e->D, b->hop, b->n_frames), s16) * sample_bytes;
        if(int rc = reserve_bytes(e, e->s_window, win))
            return rc;
        // slots that may still owe samples to the sync offset (none in steady state: no mask work then).  A captured call
        // leaves the host's counts alone: only its replays, on the device, lower them.
        e->startup = false;
        const long long L = (long long)T * b->hop;
        for(size_t s = 0; s < S; ++s)
        {
            long long &owed = e->owed[(size_t)b->first_stream + s];
            e->startup = e->startup || owed > 0;
            if(!e->capturing)
                owed = std::max(0LL, owed - L);
        }
        if(e->startup)
        {
            if(int rc = e->s_mask.reserve(e, S * T))
                return rc;
        }
    }
    // per-tick gravity (TVEXPONENTIAL only): evaluated on the host exactly as get_gravity(seconds) does, one pair per tick
    const float *d_gtab = nullptr;
    if(b->frame_seconds != nullptr && t.cfg.tsmoothing == WF_TSMOOTH_TVEXPONENTIAL)
    {
        if(int rc = e->s_gtab.reserve(e, 2 * T))
            return rc;
        e->h_gtab.resize(2 * T);
        for(size_t i = 0; i < T; ++i)
        {
            const float g = gravity_for(t.cfg, b->frame_seconds[i]);
            e->h_gtab[2 * i] = g;
            e->h_gtab[2 * i + 1] = 1.0f - g;
        }
        d_gtab = e->s_gtab;
        if(e->capturing) // the graph's own copy: its replays apply the gains it was captured with
        {
            void *d = nullptr;
            if(int rc = keep_upload(e, e->h_gtab.data(), 2 * T * sizeof(float), st, &d))
                return rc;
            d_gtab = static_cast<const float *>(d);
        }
        else
            WF_CHECK(e, cudaMemcpyAsync(e->s_gtab, e->h_gtab.data(), 2 * T * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    bool dev_ptrs = false;
    {
        // Live ticks (one source, one frame: tens of KB) in page-locked, device-mapped host buffers (wf_host_alloc) skip the
        // staging copies altogether: the kernel reads the frame and writes the spectrum over PCIe itself, so a tick costs one
        // launch + one synchronisation.  Every buffer of the batch must be device-addressable for that.
        const void *ptrs[1 + wf_engine::kBatchBufs] = {b->pcm};
        for(int i = 0; i < wf_engine::kBatchBufs; ++i)
            ptrs[1 + i] = bufs[i].of(*b);
        const bool small = S * T * (size_t)cc * (size_t)N * sample_bytes <= (1u << 20);
        if(e->zc_valid && memcmp(ptrs, e->zc_ptrs, sizeof(ptrs)) == 0)
            dev_ptrs = e->zc_dev || (e->zc_ok && small && e->knobs.zero_copy); // same buffers as the last call, already classified
        else
        {
            const int kpcm = ptr_kind(b->pcm);
            bool zc = (kpcm == 2); // every buffer device-addressable?
            for(int i = 1; i <= wf_engine::kBatchBufs && zc; ++i)
                zc = (ptrs[i] == nullptr) || (ptr_kind(ptrs[i]) != 0);
            memcpy(e->zc_ptrs, ptrs, sizeof(ptrs));
            e->zc_dev = (kpcm == 1);
            e->zc_ok = zc;
            e->zc_valid = true;
            dev_ptrs = e->zc_dev || (zc && small && e->knobs.zero_copy);
        }
    }

    if(dev_ptrs)
    {
        WF_CHECK(e, time_begin(e, st));
        if(b->out_peak)
        {
            int rc = fill_device(e, b->out_peak, (long long)T, -INFINITY, st);
            if(rc)
                return rc;
        }
        if(int rc = launch_range(e, b, bufs, st, 0, b->n_streams, d_gtab))
            return rc;
        WF_CHECK(e, time_end(e, st));
        return WF_OK;
    }

    // ---- host buffers: stage through device memory, chunked over streams so that the H2D copy of chunk i+1, the
    //      kernel of chunk i and the D2H copy of chunk i-1 overlap (PCIe is full duplex; pinned memory required for
    //      real overlap, pageable memory still works but serialises) ----
    // a ring call's stream holds only its new samples: T*hop per channel
    const size_t per_stream_span = (size_t)(cc - 1) * (size_t)b->channel_stride +
                                   (ring ? T * (size_t)b->hop : (T - 1) * (size_t)b->hop + (size_t)N);
    const size_t span = (S - 1) * (size_t)b->stream_stride + per_stream_span;
    // the batch the kernels run on: the staging buffers in place of the caller's, null where the caller passed none
    wf_batch staged = *b;
    int rc = reserve_bytes(e, e->s_pcm, span * sample_bytes);
    staged.pcm = e->s_pcm;
    for(const BatchBuf &u : bufs)
        if(u.of(*b) && !rc)
        {
            rc = reserve_bytes(e, *u.stage, u.per_stream ? S * u.bytes : u.bytes);
            u.set(staged, u.stage->p);
        }
    if(rc)
        return rc;
    if(!e->s_h2d)
    {
        WF_CHECK(e, outside_capture(e, [&] {
            cudaError_t err = cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking);
            if(!err)
                err = cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking);
            for(auto *evs : {&e->chunk_in, &e->chunk_k})
                for(auto &ev : *evs)
                    if(!err)
                        err = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
            if(!err)
                err = cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming);
            return err ? err : cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming);
        }));
    }
    const size_t in_bytes = span * sample_bytes;
    int nchunks = (int)std::min<size_t>(std::min<size_t>(wf_engine::kMaxChunks, S), std::max<size_t>(1, in_bytes >> 25));
    const int per = (int)((S + nchunks - 1) / nchunks);
    nchunks = (int)((S + per - 1) / per);

    WF_CHECK(e, time_begin(e, st));
    WF_CHECK(e, cudaEventRecord(e->ev_fork, st));
    WF_CHECK(e, cudaStreamWaitEvent(e->s_h2d, e->ev_fork, 0));
    WF_CHECK(e, cudaStreamWaitEvent(e->s_d2h, e->ev_fork, 0));
    if(staged.out_peak)
    {
        if((rc = fill_device(e, staged.out_peak, (long long)T, -INFINITY, st)))
            return rc;
    }
    for(int c = 0; c < nchunks; ++c)
    {
        const int s0 = c * per;
        const int cnt = std::min<int>(per, (int)S - s0);
        const size_t off = (size_t)s0 * (size_t)b->stream_stride;
        const size_t cspan = (size_t)(cnt - 1) * (size_t)b->stream_stride + per_stream_span;
        WF_CHECK(e, cudaMemcpyAsync(const_cast<float *>(pcm_offset(e->s_pcm, off, s16)), pcm_offset(b->pcm, off, s16),
                                   cspan * sample_bytes, cudaMemcpyHostToDevice, e->s_h2d));
        for(const BatchBuf &u : bufs)
            if(char *h = u.of(*b); h && u.in && u.per_stream)
                WF_CHECK(e, cudaMemcpyAsync(u.of(staged) + s0 * u.bytes, h + s0 * u.bytes, cnt * u.bytes,
                                           cudaMemcpyHostToDevice, e->s_h2d));
        WF_CHECK(e, cudaEventRecord(e->chunk_in[c], e->s_h2d));
        WF_CHECK(e, cudaStreamWaitEvent(st, e->chunk_in[c], 0));
        if((rc = launch_range(e, &staged, bufs, st, s0, cnt, d_gtab)))
            return rc;
        WF_CHECK(e, cudaEventRecord(e->chunk_k[c], st));
        WF_CHECK(e, cudaStreamWaitEvent(e->s_d2h, e->chunk_k[c], 0));
        for(const BatchBuf &u : bufs)
            if(char *h = u.of(*b); h && !u.in && u.per_stream)
                WF_CHECK(e, cudaMemcpyAsync(h + s0 * u.bytes, u.of(staged) + s0 * u.bytes, cnt * u.bytes,
                                           cudaMemcpyDeviceToHost, e->s_d2h));
    }
    WF_CHECK(e, time_end(e, st));
    for(const BatchBuf &u : bufs) // out_peak: complete only after the last chunk's kernel
        if(char *h = u.of(*b); h && !u.per_stream)
            WF_CHECK(e, cudaMemcpyAsync(h, u.of(staged), u.bytes, cudaMemcpyDeviceToHost, e->s_d2h));
    WF_CHECK(e, cudaEventRecord(e->ev_join, e->s_d2h));
    WF_CHECK(e, cudaStreamWaitEvent(st, e->ev_join, 0)); // the caller's stream completes when the results are home
    return WF_OK;
}

int wf_process(wf_engine *e, const wf_batch *b)
{
    int rc = wf_process_async(e, b, nullptr);
    if(rc)
        return rc;
    WF_CHECK(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

int wf_synchronize(wf_engine *e)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    WF_CHECK(e, cudaSetDevice(e->device));
    WF_CHECK(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

int wf_reset_state(wf_engine *e, int32_t first, int32_t count)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    if(int rc = check_slot_range(e, first, count, e->tab.cfg.max_streams, "reset"))
        return rc;
    if(count == 0)
        return WF_OK;
    WF_CHECK(e, cudaSetDevice(e->device));
    // on the device, per stream, so that a stream that is already silent keeps its buffers exactly as the reference's
    // early return does (src/source_generic.cpp:38-39)
    const Tables &t = e->tab;
    const bool below = !(t.db_min > (float)(t.cfg.floor_db - 10));
    const unsigned char fl = (unsigned char)(1u | (below ? 6u : 0u));
    const size_t B = (size_t)t.B;
    WF_CHECK(e, launch_kernel(spectrum_reset_kernel, e->device, std::min(count, e->sm_count * 8), 256, 0, e->stream, {},
                              e->d_state + (size_t)first * t.cfg.capture_channels * B,
                              e->d_hold + (size_t)first * t.output_channels * B, e->d_flags + first, count,
                              (int)(t.cfg.capture_channels * B), (int)(t.output_channels * B), (int)(t.display_channels * B),
                              t.db_min, fl));
    e->launches++;
    WF_CHECK(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

int wf_get_state(wf_engine *e, int32_t first, int32_t count, float *tsmooth, float *hold_db, uint8_t *flags)
{
    return spectrum_state(e, first, count, tsmooth, hold_db, flags, false);
}

int wf_get_ring(wf_engine *e, int32_t first, int32_t count, float *samples)
{
    if(int rc = ring_access(e, first, count, samples))
        return rc;
    const size_t n = (size_t)e->tab.cfg.capture_channels * (e->tab.N + e->D);
    WF_CHECK(e, cudaMemcpy(samples, e->d_ring + first * n, count * n * sizeof(float), cudaMemcpyDeviceToHost));
    return WF_OK;
}

int wf_set_ring(wf_engine *e, int32_t first, int32_t count, const float *samples)
{
    if(int rc = ring_access(e, first, count, samples))
        return rc;
    const size_t n = (size_t)e->tab.cfg.capture_channels * (e->tab.N + e->D);
    WF_CHECK(e, cudaMemcpy(e->d_ring + first * n, samples, count * n * sizeof(float), cudaMemcpyHostToDevice));
    std::fill(e->owed.begin() + first, e->owed.begin() + first + count, 0LL); // a primed stream has its delay's audio
    if(e->d_owed.p && count > 0)
    {
        WF_CHECK(e, cudaMemsetAsync(e->d_owed + first, 0, (size_t)count * sizeof(long long), e->stream));
        WF_CHECK(e, cudaStreamSynchronize(e->stream));
    }
    return WF_OK;
}

int wf_set_state(wf_engine *e, int32_t first, int32_t count, const float *tsmooth, const float *hold_db,
                 const uint8_t *flags)
{
    return spectrum_state(e, first, count, tsmooth, hold_db, flags, true);
}

int wf_peak_normalize(wf_engine *e, float *data, int32_t n_streams, int32_t n_frames, int32_t row_len,
                      const float *peak, float target_db, float max_gain, void *cuda_stream)
{
    if(!e || !data || !peak || n_streams < 0 || n_frames < 0 || row_len < 1)
        return e ? fail(e, WF_ERR_INVALID_ARG, "bad peak_normalize arguments") : WF_ERR_INVALID_ARG;
    NvtxRange nvtx("wf_peak_normalize");
    if(n_streams == 0 || n_frames == 0)
        return WF_OK;
    WF_CHECK(e, cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    WF_CHECK(e, begin_call(e, st));
    if(int rc = refuse_pageable(e, {data, peak}))
        return rc;
    const int rows_per_frame = e->tab.display_channels;
    const size_t total = (size_t)n_streams * n_frames * rows_per_frame * row_len;
    const bool dev = is_device_ptr(data);
    // host rows go through the engine's staging buffers, in and out on `st`
    Staging sg(e, st, !dev);
    float *d_data = const_cast<float *>(sg.in(e->s_out_db, static_cast<const float *>(data), total));
    Staging sp(e, st, !dev || !is_device_ptr(peak)); // a host peak is copied even with device rows
    const float *d_peak = sp.in(e->s_peak, peak, (size_t)n_frames);
    if(sp.rc)
        return sp.rc;
    sg.out(e->s_out_db, data, total);
    if(sg.rc)
        return sg.rc;
    WF_CHECK(e, time_begin(e, st));
    const long long rows = (long long)n_streams * n_frames * rows_per_frame;
    const int grid = (int)std::min<long long>(rows, (long long)e->sm_count * 16);
    WF_CHECK(e, launch_kernel(peak_normalize_kernel, e->device, grid, 256, 0, st, {}, d_data, n_streams, n_frames,
                              rows_per_frame, row_len, d_peak, target_db, max_gain));
    e->launches++;
    WF_CHECK(e, time_end(e, st));
    if(dev)
        return WF_OK;
    if(int rc = sg.finish())
        return rc;
    if(!e->capturing)
        WF_CHECK(e, cudaStreamSynchronize(st));
    return WF_OK;
}

int wf_render(wf_engine *e, const wf_render_batch *rb, void *cuda_stream)
{
    if(!e || !rb)
        return WF_ERR_INVALID_ARG;
    NvtxRange nvtx("wf_render");
    if(rb->struct_size != sizeof(wf_render_batch))
        return fail(e, WF_ERR_ABI, "wf_render_batch.struct_size %u != %zu", rb->struct_size, sizeof(wf_render_batch));
    const Tables &t = e->tab;
    const int dch = t.display_channels, B = t.B, np = t.num_points;
    if(rb->n_streams < 0 || rb->n_frames < 0)
        return fail(e, WF_ERR_INVALID_ARG, "n_streams/n_frames must be >= 0");
    const bool display = rb->out_points || rb->out_pixels || rb->out_min;
    if(display && np <= 0)
        return fail(e, WF_ERR_INVALID_ARG, "display outputs requested but the engine has no display points");
    if(rb->write_db && !rb->peak)
        return fail(e, WF_ERR_INVALID_ARG, "write_db is set but the call carries no peak");
    if(!display && !rb->write_db)
        return fail(e, WF_ERR_INVALID_ARG, "nothing requested: no display output and no write_db");
    if(rb->n_streams == 0 || rb->n_frames == 0)
        return WF_OK;
    if(!rb->db)
        return fail(e, WF_ERR_INVALID_ARG, "db is null");

    WF_CHECK(e, cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    WF_CHECK(e, begin_call(e, st));
    if(int rc = refuse_pageable(e, {rb->db, rb->peak, rb->out_points, rb->out_pixels, rb->out_min}))
        return rc;
    const size_t T = (size_t)rb->n_frames, rows = (size_t)rb->n_streams * T, n_db = rows * dch * B, n_pts = rows * dch * np;
    const bool dev = is_device_ptr(rb->db);
    KParams kp{};
    kp.n_streams = rb->n_streams;
    kp.n_frames = rb->n_frames;
    kp.dch = dch;
    set_display_params(e, kp);
    RenderArgs ra{.db = rb->db, .peak = rb->peak, .target_db = rb->target_db, .max_gain = rb->max_gain,
                  .write_db = rb->write_db ? 1 : 0, .display = display ? 1 : 0, .rows = (long long)rows, .n_frames = rb->n_frames, .B = B,
                  .len = dch * B};
    // host buffers go through the engine's staging buffers, in and out on `st`
    Staging sg(e, st, !dev);
    ra.db = const_cast<float *>(sg.in(e->s_out_db, static_cast<const float *>(rb->db), n_db));
    Staging sp(e, st, rb->peak && (!dev || !is_device_ptr(rb->peak))); // a host peak is copied even with device rows
    ra.peak = sp.in(e->s_peak, rb->peak, T);
    if(sp.rc)
        return sp.rc;
    if(rb->write_db && !dev)
        sg.out(e->s_out_db, rb->db, n_db);
    kp.out_points = sg.out(e->s_out_points, rb->out_points, n_pts);
    kp.out_pixels = sg.out(e->s_px, rb->out_pixels, n_pts);
    kp.out_min = sg.out(e->s_min, rb->out_min, rows * 2);
    if(sg.rc)
        return sg.rc;
    ra.vec4 = ((uintptr_t)ra.db & 15u) == 0;

    RenderPlan pl;
    WF_CHECK(e, render_plan(kp, B, (long long)rows, e->sm_count, e->device, &pl));
    if(pl.grid == 0)
        return fail(e, WF_ERR_INVALID_ARG, "the display stage's scratch (%d points x %d channels) exceeds shared memory", np, dch);
    ra.tab_smem = pl.tab_smem;
    ra.row_smem = pl.row_smem;
    ra.tab_floats = pl.tab_floats;
    ra.group_floats = pl.group_floats;
    if(!pl.row_smem)
    {
        if(int rc = e->s_render.reserve(e, (size_t)pl.grid * pl.groups * ra.len))
            return rc;
        ra.scratch = e->s_render;
    }
    WF_CHECK(e, time_begin(e, st));
    WF_CHECK(e, render_launch(pl, kp, ra, st, e->device));
    e->launches++;
    WF_CHECK(e, time_end(e, st));
    char name[128];
    if(pl.tn == 32)
        snprintf(name, sizeof name, "render_kernel<32> grid %d x %d warps", pl.grid, pl.groups);
    else
        snprintf(name, sizeof name, "render_kernel<%d> grid %d", pl.tn, pl.grid);
    e->last_kernel = name;
    if(dev)
        return WF_OK;
    if(int rc = sg.finish())
        return rc;
    if(!e->capturing)
        WF_CHECK(e, cudaStreamSynchronize(st));
    return WF_OK;
}

void *wf_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if(bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess)
    {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

void wf_host_free(void *p)
{
    if(p)
        cudaFreeHost(p);
}

int64_t wf_launch_count(const wf_engine *e) { return e ? e->launches : 0; }

const char *wf_last_kernel_name(const wf_engine *e) { return e ? e->last_kernel.c_str() : ""; }

float wf_last_kernel_ms(wf_engine *e) { return last_kernel_ms(e); }

} // extern "C"
