// wf_engine.cu — libwfstft.so: the C ABI of include/wfstft.h on top of the fused sm_90a kernel.
//
// Host responsibilities (mirrors what WAVSource owns in the reference, src/source.hpp:95-347):
//   * settings -> tables (wf_tables.cpp ≙ WAVSource::update), uploaded once per engine
//   * per-stream recurrence state in device memory (m_tsmooth_buf, m_decibels, m_last_silent)
//   * staging of host buffers, kernel dispatch by (fft_size, capture_channels), error reporting
// There is no CPU compute path: if CUDA is unavailable wf_create fails.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "wf_kernels.cuh"
#include "wf_fast2048.cuh"
#include "wf_anyn.cuh"
#include "wf_wide.hpp"
#include "wf_v3.hpp"
#include "wf_team2048.hpp"
#include "wf_warp2.hpp"
#include "wf_par16384.hpp"
#include "wf_nvtx.hpp"
#include "wf_tables.hpp"
#include "wfstft.h"

using namespace wf;

struct wf_engine {
    Tables tab;
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool ev_valid = false;
    std::string last_error;
    int64_t launches = 0;
    std::string last_kernel;    // name of the spectrum kernel the most recent launch_range dispatched to (wf_last_kernel_name)
    bool hold_implicit = false; // some stream may carry flags bit 3 (m_decibels mirror left implicit by the N=2048 kernel)
    bool use_par16384 = true;   // WF_PAR16384=0: N=16384 stays on the CTA-per-tick kernel (A/B tests)
    bool use_warp2_display = true; // WF_WARP2_DISPLAY=0: display outputs stay on the CTA-per-tick / any-N kernels (A/B tests)
    bool use_warp2 = true;      // WF_WARP2=0: non-power-of-two sizes stay on the first-generation any-N kernel (A/B tests)
    bool lazy_hold = true;      // WF_LAZY_HOLD=0: always write the mirror (A/B tests)
    bool split_runs = true;     // WF_SPLIT=0: whole streams per warp in the N=2048 warp-per-stream kernel (A/B tests)
    bool force_generic = false; // WF_FORCE_GENERIC=1: bypass the specialised N=2048 kernel (A/B tests)
    int fast_maxw = 16;         // WF_FAST_MAXW=12|16: which compiled variant of the N=2048 kernel (tuning knob)
    int fast_wpc_override = 0;  // WF_FAST_WPC=n: force warps per CTA (tuning knob)
    bool use_pdl = true;        // WF_NO_PDL=1: launch the fast kernel without programmatic dependent launch
    int wide_r = 0;             // WF_WIDE_R=1|2|4|8: force the cluster size of the wide kernel (1 = never use it); 0 = automatic

    // device tables
    float *d_window = nullptr, *d_slope = nullptr, *d_rolloff = nullptr;
    float *d_tw = nullptr, *d_tw_post = nullptr;
    float *d_tw1 = nullptr, *d_tw2 = nullptr, *d_tw0 = nullptr; // inter-pass twiddles of the CTA-per-tick kernel (wf_v3.cuh), N = 4096/8192/16384
    // N=2048: the warp-per-stream kernel needs ~2400 streams to fill the GPU; with fewer streams AND long per-stream tick
    // sequences (>= 32) the cluster kernel (wf_v3.cuh, up to 8 ticks of a stream in flight) is faster: measured 256x256
    // 96 -> 145 M, 512x128 185 -> 202 M, 1024x64 286 vs 242 M spectra/s (profiles/r01_layouts.txt).  WF_FAST_MIN_STREAMS overrides.
    int fast_min_streams = 768;
    int team_w = 0;                            // WF_TEAM_W=4|8|16: force the team size of wf_team2048.cuh; 1: never use it; 0 = automatic
    bool use_v3 = true;                        // WF_V3=0: fall back to the first-generation kernels (A/B tests)
    float *d_interp_idx = nullptr, *d_interp_w = nullptr, *d_gauss = nullptr;
    int *d_band_widths = nullptr, *d_band_offsets = nullptr;
    // per-stream state
    float *d_state = nullptr, *d_hold = nullptr;
    unsigned char *d_flags = nullptr;
    // staging for host-pointer batches (grown on demand)
    float *s_pcm = nullptr, *s_out_db = nullptr, *s_out_points = nullptr, *s_rms = nullptr, *s_peak = nullptr;
    unsigned char *s_skip = nullptr, *s_silent = nullptr;
    float *s_px = nullptr, *s_min = nullptr;
    float *s_gtab = nullptr; // [n_frames][2] per-tick (g, 1-g) of a TV-exponential batch with frame_seconds
    size_t s_gtab_cap = 0;
    std::vector<float> h_gtab;
    size_t s_px_cap = 0, s_min_cap = 0;
    float *s_scratch = nullptr; // any-N kernel work buffers when N/2 complex points x 2 exceed shared memory
    size_t s_scratch_cap = 0;
    size_t s_pcm_cap = 0, s_out_db_cap = 0, s_out_points_cap = 0, s_rms_cap = 0, s_peak_cap = 0, s_skip_cap = 0,
           s_silent_cap = 0;
    // zero-copy verdict of the last host-pointer batch (live ticks reuse the same buffers every call)
    const void *zc_ptrs[9] = {};
    bool zc_ok = false, zc_dev = false, zc_valid = false;
    bool zero_copy = true; // WF_ZERO_COPY=0: always stage host buffers through device memory
    // copy/compute pipeline for host-pointer batches
    static constexpr int kMaxChunks = 16;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t chunk_in[kMaxChunks] = {}, chunk_k[kMaxChunks] = {}, ev_fork = nullptr, ev_join = nullptr;
};

namespace {

thread_local std::string g_create_error;

int set_err(wf_engine *e, int code, const char *fmt, ...)
{
    if(e)
    {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof(buf), fmt, ap);
        va_end(ap);
        e->last_error = buf;
    }
    return code;
}

#define WF_CUDA(e, call)                                                                                              \
    do                                                                                                                \
    {                                                                                                                 \
        cudaError_t _err = (call);                                                                                    \
        if(_err != cudaSuccess)                                                                                       \
            return set_err((e), (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s failed: %s", #call, \
                           cudaGetErrorString(_err));                                                                 \
    } while(0)

template<typename T>
int upload(wf_engine *e, T **dst, const std::vector<T> &src)
{
    *dst = nullptr;
    if(src.empty())
        return WF_OK;
    WF_CUDA(e, cudaMalloc((void **)dst, src.size() * sizeof(T)));
    WF_CUDA(e, cudaMemcpy(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
    return WF_OK;
}

template<typename T>
int ensure(wf_engine *e, T **buf, size_t *cap, size_t need)
{
    if(need <= *cap)
        return WF_OK;
    if(*buf)
        cudaFree(*buf);
    *buf = nullptr;
    *cap = 0;
    WF_CUDA(e, cudaMalloc((void **)buf, need * sizeof(T)));
    *cap = need;
    return WF_OK;
}

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

// 0 = pageable host (or unknown), 1 = device / managed, 2 = page-locked host memory the device can address directly
int ptr_kind(const void *p)
{
    cudaPointerAttributes a{};
    if(cudaPointerGetAttributes(&a, p) != cudaSuccess)
    {
        cudaGetLastError();
        return 0;
    }
    if(a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)
        return 1;
    if(a.type == cudaMemoryTypeHost && a.devicePointer == p) // unified addressing: the same pointer is valid on the device
        return 2;
    return 0;
}

bool is_device_ptr(const void *p)
{
    if(!p)
        return false;
    cudaPointerAttributes a{};
    if(cudaPointerGetAttributes(&a, p) != cudaSuccess)
    {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

template<int N, int CC>
int launch_fused(wf_engine *e, const KParams &kp, cudaStream_t st, size_t extra_smem)
{
    using G = Geo<N>;
    const size_t smem = (size_t)G::GROUPS * G::BUF * sizeof(float2) + extra_smem;
    static thread_local size_t configured[64] = {0};
    int dev = e->device & 63;
    if(smem > 48 * 1024 && configured[dev] < smem)
    {
        WF_CUDA(e, cudaFuncSetAttribute(stft_fused_kernel<N, CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[dev] = smem;
    }
    const int grid = (kp.n_streams + G::GROUPS - 1) / G::GROUPS;
    stft_fused_kernel<N, CC><<<grid, G::CTA, smem, st>>>(kp);
    WF_CUDA(e, cudaGetLastError());
    e->launches++;
    e->last_kernel = "stft_fused_kernel<" + std::to_string(N) + "," + std::to_string(CC) + ">";
    return WF_OK;
}

// Cluster size of the wide kernel (wf_wide.cuh) for this launch, 1 = use the one-group-per-stream kernel.
// The wide kernel pays off when there are too few streams to fill the GPU: R CTAs per stream work on R ticks at once.
int pick_wide_r(const wf_engine *e, const KParams &kp, bool display)
{
    const int N = e->tab.N;
    if(!wide_supported(N) || e->wide_r == 1)
        return 1;
    if(wide_smem_bytes(N, kp.dch, kp.scratch_q, display) > 227 * 1024)
        return 1;
    if(e->wide_r == 2 || e->wide_r == 4 || e->wide_r == 8)
        return e->wide_r;
    int r = 1;
    while(r < 8 && (long long)kp.n_streams * r < 2LL * e->sm_count && 2 * r <= kp.n_frames)
        r *= 2;
    return r;
}

// Cluster size for the CTA-per-tick kernel (wf_v3.cuh): 1 when the streams alone fill the GPU, else up to 8 CTAs
// (= 8 ticks in flight) per stream.
int pick_v3_r(const wf_engine *e, const KParams &kp)
{
    const int rmin = v3_min_cluster(e->tab.N);
    if(e->wide_r == 1 || e->wide_r == 2 || e->wide_r == 4 || e->wide_r == 8)
        return std::max(rmin, e->wide_r);
    int r = rmin;
    while(r < 8 && (long long)kp.n_streams * r * 3 < 5LL * e->sm_count && 2 * r <= kp.n_frames) // per-tick overhead grows with R
        r *= 2;
    return r;
}

template<int CC>
int dispatch_n(wf_engine *e, const KParams &kp, cudaStream_t st, size_t extra)
{
    {
        const bool display = kp.out_points || kp.out_pixels || kp.out_min;
        if(e->use_v3 && e->d_tw1 != nullptr && v3_smem_bytes(e->tab.N, kp.dch, kp.scratch_q, display, CC, 8) <= 227 * 1024)
        {
            const bool feat = kp.slope || kp.rolloff || kp.normalize || kp.fast_peaks || kp.skip_mask || kp.g_tab;
            const int x = feat ? 3 : (kp.out_peak ? 1 : 0);
            const int r = pick_v3_r(e, kp);
            WF_CUDA(e, v3_launch(e->tab.N, CC, r, x, kp, e->d_tw1, e->d_tw2, e->d_tw0, st, display, e->device));
            e->launches++;
            e->last_kernel = "stft_v3_kernel<" + std::to_string(e->tab.N) + "," + std::to_string(CC) + "," + std::to_string(r) +
                             "," + std::to_string(x) + ">";
            return WF_OK;
        }
        const int R = pick_wide_r(e, kp, display);
        if(R > 1)
        {
            WF_CUDA(e, wide_launch(e->tab.N, CC, R, kp, st, display, e->device));
            e->launches++;
            e->last_kernel = "stft_wide_kernel<" + std::to_string(e->tab.N) + "," + std::to_string(CC) + "," + std::to_string(R) + ">";
            return WF_OK;
        }
    }
    switch(e->tab.N)
    {
    case 128: return launch_fused<128, CC>(e, kp, st, extra);
    case 256: return launch_fused<256, CC>(e, kp, st, extra);
    case 512: return launch_fused<512, CC>(e, kp, st, extra);
    case 1024: return launch_fused<1024, CC>(e, kp, st, extra);
    case 2048: return launch_fused<2048, CC>(e, kp, st, extra);
    case 4096: return launch_fused<4096, CC>(e, kp, st, extra);
    case 8192: return launch_fused<8192, CC>(e, kp, st, extra);
    case 16384: return launch_fused<16384, CC>(e, kp, st, extra);
    case 32768: return launch_fused<32768, CC>(e, kp, st, extra);
    default: break;
    }
    // any other multiple of 16: run-time mixed-radix kernel
    AnyPlan plan;
    if(!make_any_plan(e->tab.N, &plan))
        return set_err(e, WF_ERR_UNSUPPORTED_FFT_SIZE, "fft_size %d has no kernel", e->tab.N);
    const bool in_smem = (size_t)plan.M * 16 + extra <= 200 * 1024;
    int grid = std::min(kp.n_streams, e->sm_count * (in_smem ? 8 : 2));
    size_t smem = in_smem ? (size_t)plan.M * 16 + extra : extra;
    plan.scratch = nullptr;
    if(!in_smem)
    {
        int rc = ensure(e, &e->s_scratch, &e->s_scratch_cap, (size_t)grid * 2 * plan.M * 2);
        if(rc)
            return rc;
        plan.scratch = reinterpret_cast<float2 *>(e->s_scratch);
    }
    static thread_local size_t configured[64] = {0};
    const int dev = e->device & 63;
    if(smem > 48 * 1024 && configured[dev] < smem)
    {
        WF_CUDA(e, cudaFuncSetAttribute(stft_anyn_kernel<CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[dev] = smem;
    }
    stft_anyn_kernel<CC><<<grid, kAnyThreads, smem, st>>>(kp, plan);
    WF_CUDA(e, cudaGetLastError());
    e->launches++;
    e->last_kernel = "stft_anyn_kernel<" + std::to_string(CC) + "> N=" + std::to_string(e->tab.N);
    return WF_OK;
}

// One CTA per SM; the kernel deals streams round-robin to CTAs first, so each SM gets n_streams/grid (+-1) whole
// streams (the unit of work: EMA state stays on-chip across a stream's frames) and runs min(max_wpc, that) warps.
static void fast2048_geometry(int n_streams, int sm_count, int max_wpc, int *warps_per_cta, int *grid)
{
    *grid = std::min(n_streams, sm_count);
    const int per_cta = (n_streams + *grid - 1) / *grid;
    // at least 8 warps even for one stream: the CTA prologue (tables -> shared memory) is spread over the CTA's threads, and
    // with a single warp it dominated the latency of a live tick (1 stream x 1 frame: 19.7 -> ~8 us of kernel time)
    *warps_per_cta = std::max(std::min(8, max_wpc), std::min(max_wpc, per_cta));
}

template<int MAXW, bool TSM, bool GATE, bool EXTRA>
int launch_fast2048(wf_engine *e, const KParams &kp, cudaStream_t st)
{
    static thread_local bool configured[64] = {false};
    const int dev = e->device & 63;
    if(!configured[dev])
    {
        WF_CUDA(e, cudaFuncSetAttribute(stft2048_fast_kernel<MAXW, TSM, GATE, EXTRA>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, fast::smem_bytes(MAXW)));
        configured[dev] = true;
    }
    int wpc = MAXW, grid = 1;
    fast2048_geometry(kp.n_streams, e->sm_count, MAXW, &wpc, &grid);
    if(e->fast_wpc_override > 0 && e->fast_wpc_override <= MAXW)
    {
        wpc = e->fast_wpc_override;
        grid = std::min(kp.n_streams, e->sm_count);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)(wpc * 32));
    cfg.dynamicSmemBytes = fast::smem_bytes(wpc);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; // PDL: prologue overlaps the previous launch's tail
    attr[0].val.programmaticStreamSerializationAllowed = e->use_pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    WF_CUDA(e, cudaLaunchKernelEx(&cfg, stft2048_fast_kernel<MAXW, TSM, GATE, EXTRA>, kp));
    e->launches++;
    e->last_kernel = "stft2048_fast_kernel<" + std::to_string(MAXW) + "," + std::to_string((int)TSM) + "," + std::to_string((int)GATE) +
                     "," + std::to_string((int)EXTRA) + "> grid " + std::to_string(grid) + " x " + std::to_string(wpc) + " warps";
    return WF_OK;
}


// Hand-specialised path for the headline shape (see wf_fast2048.cuh); everything else takes the generic kernel.
int dispatch_fast2048(wf_engine *e, const KParams &kp, cudaStream_t st, bool extra)
{
    const bool tsm = kp.tsmooth != 0, gate = kp.gate != 0;
    const int maxw = e->fast_maxw;
#define WF_FAST_CASE(W, T, G, X)            \
    if(maxw == W && tsm == T && gate == G && extra == X) \
        return launch_fast2048<W, T, G, X>(e, kp, st);
    WF_FAST_CASE(16, true, true, false)
    WF_FAST_CASE(16, true, true, true)
    WF_FAST_CASE(16, true, false, false)
    WF_FAST_CASE(16, true, false, true)
    WF_FAST_CASE(16, false, true, false)
    WF_FAST_CASE(16, false, true, true)
    WF_FAST_CASE(16, false, false, false)
    WF_FAST_CASE(16, false, false, true)
    WF_FAST_CASE(12, true, true, false)
    WF_FAST_CASE(12, true, true, true)
    WF_FAST_CASE(12, true, false, false)
    WF_FAST_CASE(12, true, false, true)
    WF_FAST_CASE(12, false, true, false)
    WF_FAST_CASE(12, false, true, true)
    WF_FAST_CASE(12, false, false, false)
    WF_FAST_CASE(12, false, false, true)
#undef WF_FAST_CASE
    return set_err(e, WF_ERR_INVALID_ARG, "fast2048 dispatch fell through");
}

int fill_device(wf_engine *e, float *p, long long n, float v, cudaStream_t st)
{
    if(n <= 0)
        return WF_OK;
    int blocks = (int)std::min<long long>((n + 255) / 256, 1184);
    fill_kernel<<<blocks, 256, 0, st>>>(p, n, v);
    WF_CUDA(e, cudaGetLastError());
    e->launches++;
    return WF_OK;
}

// Write out every implicit m_decibels mirror (see materialize_hold_kernel) before something other than the N=2048
// warp-per-stream kernel looks at hold_db.
int materialize_hold(wf_engine *e, cudaStream_t st)
{
    if(!e->hold_implicit)
        return WF_OK;
    const Tables &t = e->tab;
    const int S = t.cfg.max_streams;
    materialize_hold_kernel<<<std::min(S, e->sm_count * 8), 256, 0, st>>>(e->d_state, e->d_hold, e->d_flags, S, t.B,
                                                                          t.output_channels, t.db_min);
    WF_CUDA(e, cudaGetLastError());
    e->launches++;
    e->hold_implicit = false;
    return WF_OK;
}

// Fresh streams (wf_create): m_tsmooth_buf = 0, m_decibels = DB_MIN, m_last_silent = false (src/source.cpp:1176-1180, 1236).
int init_state(wf_engine *e, int first, int count, cudaStream_t st)
{
    const Tables &t = e->tab;
    const int cc = t.cfg.capture_channels, och = t.output_channels, B = t.B;
    WF_CUDA(e, cudaMemsetAsync(e->d_state + (size_t)first * cc * B, 0, (size_t)count * cc * B * sizeof(float), st));
    int rc = fill_device(e, e->d_hold + (size_t)first * och * B, (long long)count * och * B, t.db_min, st);
    if(rc)
        return rc;
    // flags: bit0 last_silent; bit1/2: previous outputs all <= floor-10 (DB_MIN is)
    const bool below = !(t.db_min > (float)(t.cfg.floor_db - 10));
    WF_CUDA(e, cudaMemsetAsync(e->d_flags + first, below ? 6 : 0, (size_t)count, st));
    return WF_OK;
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
}

int wf_create(const wf_config *cfg, wf_engine **out)
{
    if(!cfg || !out)
        return WF_ERR_INVALID_ARG;
    *out = nullptr;
    if(cfg->struct_size != sizeof(wf_config))
        return WF_ERR_ABI;
    wf_engine *e = new(std::nothrow) wf_engine();
    if(!e)
        return WF_ERR_OOM;
    auto bail = [&](int code) {
        g_create_error = e->last_error; // readable through wf_last_error(NULL) after the engine is gone
        wf_destroy(e);
        return code;
    };

    const char *why = nullptr;
    int rc = build_tables(*cfg, e->tab, &why);
    if(rc != WF_OK)
    {
        set_err(e, rc, "%s", why ? why : "bad config");
        return bail(rc);
    }
    if(!supported_fft_size(e->tab.N))
        return bail(set_err(e, WF_ERR_UNSUPPORTED_FFT_SIZE, "fft_size %d unsupported", e->tab.N));

    int ndev = 0;
    if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    {
        cudaGetLastError();
        return bail(set_err(e, WF_ERR_NO_DEVICE, "no CUDA device"));
    }
    int dev = cfg->device;
    if(dev < 0)
    {
        if(cudaGetDevice(&dev) != cudaSuccess)
            return bail(set_err(e, WF_ERR_CUDA, "cudaGetDevice failed"));
    }
    if(dev >= ndev)
        return bail(set_err(e, WF_ERR_INVALID_ARG, "device %d out of range (%d devices)", dev, ndev));
    e->device = dev;
    {
        const char *fg = getenv("WF_FORCE_GENERIC");
        e->force_generic = fg && fg[0] == '1';
        const char *mw = getenv("WF_FAST_MAXW");
        if(mw && (atoi(mw) == 12 || atoi(mw) == 16))
            e->fast_maxw = atoi(mw);
        const char *np = getenv("WF_NO_PDL");
        e->use_pdl = !(np && np[0] == '1');
        const char *wr = getenv("WF_WIDE_R");
        if(wr)
            e->wide_r = atoi(wr);
        const char *fms = getenv("WF_FAST_MIN_STREAMS");
        if(fms)
            e->fast_min_streams = atoi(fms);
        const char *v3 = getenv("WF_V3");
        e->use_v3 = !(v3 && v3[0] == '0');
        const char *tw = getenv("WF_TEAM_W");
        if(tw)
            e->team_w = atoi(tw);
        const char *zc = getenv("WF_ZERO_COPY");
        e->zero_copy = !(zc && zc[0] == '0');
        const char *p16 = getenv("WF_PAR16384");
        e->use_par16384 = !(p16 && p16[0] == '0');
        const char *w2 = getenv("WF_WARP2");
        e->use_warp2 = !(w2 && w2[0] == '0');
        const char *w2d = getenv("WF_WARP2_DISPLAY");
        e->use_warp2_display = !(w2d && w2d[0] == '0');
        const char *lh = getenv("WF_LAZY_HOLD");
        e->lazy_hold = !(lh && lh[0] == '0');
        const char *sp = getenv("WF_SPLIT");
        e->split_runs = !(sp && sp[0] == '0');
        const char *wo = getenv("WF_FAST_WPC");
        if(wo)
            e->fast_wpc_override = atoi(wo);
    }

#define WF_TRY(x)                 \
    do                            \
    {                             \
        int _rc = (x);            \
        if(_rc != WF_OK)          \
            return bail(_rc);     \
    } while(0)
#define WF_CUDA_C(call)                                                                                      \
    do                                                                                                       \
    {                                                                                                        \
        cudaError_t _err = (call);                                                                           \
        if(_err != cudaSuccess)                                                                              \
            return bail(set_err(e, (_err == cudaErrorMemoryAllocation) ? WF_ERR_OOM : WF_ERR_CUDA, "%s: %s", \
                                #call, cudaGetErrorString(_err)));                                           \
    } while(0)

    WF_CUDA_C(cudaSetDevice(dev));
    cudaDeviceProp prop{};
    WF_CUDA_C(cudaGetDeviceProperties(&prop, dev));
    e->sm_count = prop.multiProcessorCount;
    if(prop.major != 9 || prop.minor != 0) // sm_90a code runs on compute capability 9.0 only
        return bail(set_err(e, WF_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev,
                            prop.major, prop.minor));
    WF_CUDA_C(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    WF_CUDA_C(cudaEventCreate(&e->ev0));
    WF_CUDA_C(cudaEventCreate(&e->ev1));

    const Tables &t = e->tab;
    WF_TRY(upload(e, &e->d_window, t.window));
    WF_TRY(upload(e, &e->d_slope, t.slope));
    WF_TRY(upload(e, &e->d_rolloff, t.rolloff));
    WF_TRY(upload(e, &e->d_tw, t.tw));
    WF_TRY(upload(e, &e->d_tw_post, t.tw_post));
    if(v3_supported(t.N))
    {
        std::vector<float> tw1, tw2, tw0;
        v3_build_twiddles(t.N, tw1, tw2, tw0);
        WF_TRY(upload(e, &e->d_tw1, tw1));
        WF_TRY(upload(e, &e->d_tw2, tw2));
        WF_TRY(upload(e, &e->d_tw0, tw0));
    }
    WF_TRY(upload(e, &e->d_interp_idx, t.interp_indices));
    WF_TRY(upload(e, &e->d_interp_w, t.interp_weights));
    WF_TRY(upload(e, &e->d_gauss, t.gauss));
    WF_TRY(upload(e, &e->d_band_widths, t.band_widths));
    WF_TRY(upload(e, &e->d_band_offsets, t.band_offsets));

    const size_t S = (size_t)t.cfg.max_streams;
    WF_CUDA_C(cudaMalloc((void **)&e->d_state, S * t.cfg.capture_channels * t.B * sizeof(float)));
    WF_CUDA_C(cudaMalloc((void **)&e->d_hold, S * t.output_channels * t.B * sizeof(float)));
    WF_CUDA_C(cudaMalloc((void **)&e->d_flags, S));
    WF_TRY(init_state(e, 0, (int)S, e->stream));
    WF_CUDA_C(cudaStreamSynchronize(e->stream));
#undef WF_TRY
#undef WF_CUDA_C
    *out = e;
    return WF_OK;
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
    void *ptrs[] = {e->d_window, e->d_slope, e->d_rolloff, e->d_tw, e->d_tw_post, e->d_tw1, e->d_tw2, e->d_tw0, e->d_interp_idx, e->d_interp_w,
                    e->d_gauss, e->d_band_widths, e->d_band_offsets, e->d_state, e->d_hold, e->d_flags, e->s_pcm,
                    e->s_out_db, e->s_out_points, e->s_rms, e->s_peak, e->s_skip, e->s_silent, e->s_scratch, e->s_px, e->s_min, e->s_gtab};
    for(void *p : ptrs)
        if(p)
            cudaFree(p);
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
    if(e->ev0)
        cudaEventDestroy(e->ev0);
    if(e->ev1)
        cudaEventDestroy(e->ev1);
    if(e->stream)
        cudaStreamDestroy(e->stream);
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
    if(cfg->struct_size != sizeof(wf_config))
        return WF_ERR_ABI;
    Tables t;
    const char *why = nullptr;
    int rc = build_tables(*cfg, t, &why);
    if(rc != WF_OK)
    {
        g_create_error = why ? why : "bad config";
        return rc;
    }
    if(info)
        fill_info(t, info, -1, -1);
    return copy_table(t, which, out, capacity);
}

// Launch the fused kernel for streams [s0, s0+count) of the batch; all pointers are DEVICE pointers already
// offset to stream 0 of the batch.
static int launch_range(wf_engine *e, const wf_batch *b, cudaStream_t st, int s0, int count, const float *pcm,
                        const float *rms, const unsigned char *skip, float *out_db, float *out_points,
                        unsigned char *silent, float *out_peak, float *px_dev, float *min_dev, const float *g_tab_dev)
{
    const Tables &t = e->tab;
    const int cc = t.cfg.capture_channels, dch = t.display_channels, och = t.output_channels, B = t.B, N = t.N;
    const size_t T = (size_t)b->n_frames;
    KParams kp{};
    kp.pcm = pcm + (size_t)s0 * (size_t)b->stream_stride;
    kp.stream_stride = b->stream_stride;
    kp.channel_stride = b->channel_stride;
    kp.n_streams = count;
    kp.n_frames = b->n_frames;
    kp.hop = b->hop;
    kp.aligned8 = (((uintptr_t)kp.pcm & 7u) == 0) && ((b->stream_stride & 1) == 0) && ((b->channel_stride & 1) == 0) &&
                  ((b->hop & 1) == 0);
    kp.input_rms = rms ? rms + (size_t)s0 * T : nullptr;
    kp.skip_mask = skip ? skip + (size_t)s0 * T : nullptr;
    kp.window = e->d_window;
    kp.window2 = reinterpret_cast<const float2 *>(e->d_window);
    kp.tw = reinterpret_cast<const float2 *>(e->d_tw);
    kp.tw_post = reinterpret_cast<const float2 *>(e->d_tw_post);
    kp.slope = e->d_slope;
    kp.rolloff = e->d_rolloff;
    const size_t slot = (size_t)b->first_stream + (size_t)s0;
    kp.state = e->d_state + slot * cc * B;
    kp.hold_db = e->d_hold + slot * och * B;
    kp.flags = e->d_flags + slot;
    kp.out_db = out_db ? out_db + (size_t)s0 * T * dch * B : nullptr;
    kp.out_points = out_points ? out_points + (size_t)s0 * T * dch * t.num_points : nullptr;
    kp.out_silent = silent ? silent + (size_t)s0 * T : nullptr;
    kp.out_peak = out_peak;
    kp.coef_half = (2.0f / t.window_sum) * 0.5f; // mag_coefficient/2: the split pass leaves 2*X (src/source_generic.cpp:110)
    kp.g = (t.cfg.tsmoothing == WF_TSMOOTH_NONE) ? 0.0f : gravity_for(t.cfg, b->seconds);
    kp.g2 = 1.0f - kp.g;
    kp.g_tab = reinterpret_cast<const float2 *>(g_tab_dev);
    kp.tsmooth = t.cfg.tsmoothing != WF_TSMOOTH_NONE;
    kp.fast_peaks = t.cfg.fast_peaks;
    kp.stereo = t.cfg.stereo;
    kp.och = och;
    kp.dch = dch;
    kp.gate = t.cfg.silence_gate;
    kp.floor_m10 = (float)(t.cfg.floor_db - 10);
    kp.db_min = t.db_min;
    kp.normalize = t.cfg.normalize_volume;
    kp.vol_target = t.cfg.volume_target;
    kp.max_gain = t.cfg.max_gain;
    kp.write_hold = 1;
    kp.interp_idx = e->d_interp_idx;
    kp.interp_w = e->d_interp_w;
    kp.band_widths = e->d_band_widths;
    kp.band_offsets = e->d_band_offsets;
    kp.n_points = t.num_points;
    kp.n_sample = (t.cfg.display_mode == WF_DISPLAY_BAR && t.cfg.interp_mode != WF_INTERP_POINT) ? (int)t.interp_indices.size() : 0;
    kp.scratch_q = t.num_points + (dch * kp.n_sample + 3) / 4;
    kp.taps = t.interp_taps;
    kp.radius = t.interp_radius;
    kp.display_bar = (t.cfg.display_mode == WF_DISPLAY_BAR);
    kp.interp_mode = t.cfg.interp_mode;
    kp.gauss_w = e->d_gauss;
    kp.gauss_radius = t.gauss_radius;
    kp.gauss_size = (int)t.gauss.size();
    kp.gauss_sum = t.gauss_sum;
    kp.filter = (t.cfg.filter_mode == WF_FILTER_GAUSS);
    kp.out_pixels = b->out_pixels ? px_dev + (size_t)s0 * T * dch * t.num_points : nullptr;
    kp.out_min = b->out_min ? min_dev + (size_t)s0 * T * 2 : nullptr;
    kp.px_lo = t.px_lo;
    kp.px_hi = t.px_hi;
    kp.px_cpos = t.px_cpos;
    kp.ceiling_f = (float)t.cfg.ceiling_db;
    kp.dbrange_f = (float)(t.cfg.ceiling_db - t.cfg.floor_db);
    kp.mirror = t.cfg.mirror_freq_axis;

    // shared memory for the display stage: [groups][2][dch <= 2][num_points] floats
    size_t extra = 0;
    if(kp.out_points || kp.out_pixels || kp.out_min)
    {
        int groups = 1;
        switch(N)
        {
        case 128: groups = Geo<128>::GROUPS; break;
        case 256: groups = Geo<256>::GROUPS; break;
        case 512: groups = Geo<512>::GROUPS; break;
        case 1024: groups = Geo<1024>::GROUPS; break;
        case 2048: groups = Geo<2048>::GROUPS; break;
        default: groups = 1; break;
        }
        extra = (size_t)groups * 4 * (size_t)kp.scratch_q * sizeof(float);
    }
    const bool aligned16 = (((uintptr_t)kp.pcm & 15u) == 0) && ((b->stream_stride & 3) == 0) && ((b->hop & 3) == 0);
    const bool fast_ok = (N == 2048) && (cc == 1) && !t.cfg.stereo && kp.out_db && !kp.out_points && !kp.out_pixels &&
                         !kp.out_min && aligned16 && !e->force_generic;
    if(fast_ok)
    {
        const bool x = kp.slope || kp.rolloff || kp.normalize || kp.fast_peaks || kp.skip_mask || kp.out_peak || kp.g_tab;
        kp.lazy_hold = e->lazy_hold ? 1 : 0;
        kp.split = e->split_runs ? 1 : 0;
        if(kp.lazy_hold)
            e->hold_implicit = true;
        // Fewer streams than SMs x 16 warps: a team of W warps per stream works on W ticks at once (wf_team2048.cuh).
        // Up to 8 streams per SM: 16 / W = 1, 2 or 4 teams per SM (a team takes its streams one after the other); measured
        // (profiles/r02_layouts.txt) 256 x 256: 142 -> 272 M spectra/s, 512 x 128: 200 -> 310 M, 1024 x 64: 289 -> 332 M.
        int W = 1;
        if(e->team_w != 1)
        {
            const int per_sm = (kp.n_streams + e->sm_count - 1) / e->sm_count;
            if(per_sm <= 8)
                W = (per_sm <= 1) ? 16 : (per_sm == 2) ? 8 : 4;
            if(e->team_w == 4 || e->team_w == 8 || e->team_w == 16)
                W = e->team_w;
            while(W > 1 && W > kp.n_frames)
                W /= 2;
            if(W == 2)
                W = 1;
        }
        if(W > 1)
        {
            const int tpc = 16 / W;
            const int grid = std::min(e->sm_count, kp.n_streams); // streams are dealt to SMs first, then to an SM's teams
            WF_CUDA(e, team2048_launch(W, x, kp, grid, st, e->use_pdl, e->device));
            e->launches++;
            e->last_kernel = "stft2048_team_kernel<" + std::to_string(W) + "," + std::to_string((int)x) + "> grid " + std::to_string(grid) +
                             " x " + std::to_string(tpc) + " teams";
            return WF_OK;
        }
        return dispatch_fast2048(e, kp, st, x);
    }
    {
        const int rc = materialize_hold(e, st); // the other kernels read hold_db as it is
        if(rc)
            return rc;
    }
    // N = 16384 (config 5): a cluster of two CTAs per stream splits the bins by parity, each on the spill-free N=8192 plan
    const bool par_ok = (N == 16384) && e->use_par16384 && e->use_v3 && e->d_tw0 && (cc == 1) && !t.cfg.stereo && kp.out_db &&
                        !kp.out_points && !kp.out_pixels && !kp.out_min && !e->force_generic;
    if(par_ok)
    {
        const bool x = kp.slope || kp.rolloff || kp.normalize || kp.fast_peaks || kp.skip_mask || kp.out_peak || kp.g_tab;
        WF_CUDA(e, par16384_launch(x, kp, e->d_tw1, e->d_tw2, e->d_tw0, st, e->device));
        e->launches++;
        e->last_kernel = "stft16384_parity_kernel<" + std::to_string((int)x) + "> " + std::to_string(kp.n_streams) + " clusters of 2";
        return WF_OK;
    }
    // Non-power-of-two sizes with a compiled two-pass plan (wf_warp2.cuh): same launch shape as the N=2048 kernel.  With
    // display outputs (curve points / bars / pixels / minimum) the same kernel runs the render-time stages per warp; that
    // variant also takes the power-of-two sizes 512 / 1024 / 2048 (config 1: N=1024, 26 bars).
    const bool disp = kp.out_points || kp.out_pixels || kp.out_min;
    const bool warp2_ok = e->use_warp2 && (cc == 1) && !t.cfg.stereo && aligned16 &&
                          (disp ? (e->use_warp2_display && !e->force_generic && (warp2_supported(N) || warp2_pow2_supported(N)))
                                : (warp2_supported(N) && kp.out_db));
    if(warp2_ok)
    {
        const bool x = kp.slope || kp.rolloff || kp.normalize || kp.fast_peaks || kp.skip_mask || kp.out_peak || kp.g_tab;
        int wpc = 16, grid = 1;
        fast2048_geometry(kp.n_streams, e->sm_count, 16, &wpc, &grid);
        kp.split = e->split_runs ? 1 : 0;
        if(disp)
        {
            // shared memory of the display variant (layout in wf_warp2.cuh): per CTA the setup tables, per warp the tick's dB
            // row, the bar sample points and — only for the Gaussian / pixel / minimum outputs — two rows of points + scratch
            const size_t tab = display_table_floats(kp);
            const bool need_pts = kp.filter || kp.out_pixels || kp.out_min;
            const size_t per_warp = (size_t)B + (size_t)kp.n_sample + (need_pts ? 2 * (size_t)kp.n_points + 64 : 0);
            kp.disp_tab_bytes = (int)((tab * sizeof(float) + 127) / 128 * 128);
            kp.disp_bytes = (int)((per_warp * sizeof(float) + 127) / 128 * 128);
        }
        const char *name = "";
        const cudaError_t rc = warp2_launch(N, x, disp, kp, grid, &wpc, st, e->use_pdl, e->device, &name);
        if(rc != cudaErrorInvalidConfiguration) // (a curve too long for one warp's share of shared memory falls through)
        {
            WF_CUDA(e, rc);
            e->launches++;
            e->last_kernel = std::string(name) + " N=" + std::to_string(N) + " grid " + std::to_string(grid) + " x " + std::to_string(wpc) + " warps";
            return WF_OK;
        }
    }
    return (cc == 2) ? dispatch_n<2>(e, kp, st, extra) : dispatch_n<1>(e, kp, st, extra);
}

int wf_process_async(wf_engine *e, const wf_batch *b, void *cuda_stream)
{
    if(!e || !b)
        return WF_ERR_INVALID_ARG;
    NvtxRange nvtx("wf_process");
    if(b->struct_size != sizeof(wf_batch))
        return set_err(e, WF_ERR_ABI, "wf_batch.struct_size %u != %zu", b->struct_size, sizeof(wf_batch));
    const Tables &t = e->tab;
    const int cc = t.cfg.capture_channels, dch = t.display_channels, B = t.B, N = t.N;
    if(b->n_streams < 0 || b->n_frames < 0 || b->hop < 1)
        return set_err(e, WF_ERR_INVALID_ARG, "n_streams/n_frames must be >= 0 and hop >= 1");
    if(b->first_stream < 0 || (int64_t)b->first_stream + b->n_streams > t.cfg.max_streams)
        return set_err(e, WF_ERR_CAPACITY, "streams [%d, %d) exceed max_streams %d", b->first_stream,
                       b->first_stream + b->n_streams, t.cfg.max_streams);
    if(b->n_streams == 0 || b->n_frames == 0)
        return WF_OK;
    if(!b->pcm)
        return set_err(e, WF_ERR_INVALID_ARG, "pcm is null");
    if(b->stream_stride < 0 || b->channel_stride < 0)
        return set_err(e, WF_ERR_INVALID_ARG, "negative strides are not supported");
    if(t.cfg.normalize_volume && !b->input_rms)
        return set_err(e, WF_ERR_INVALID_ARG, "normalize_volume is set but the batch carries no input_rms (m_input_rms per tick: "
                                              "wf_meter in WF_METER_INPUT_RMS mode, or the host's own update_input_rms)");
    if((b->out_points || b->out_pixels || b->out_min) && t.num_points <= 0)
        return set_err(e, WF_ERR_INVALID_ARG, "display outputs requested but the engine has no display points");

    WF_CUDA(e, cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    const size_t S = (size_t)b->n_streams, T = (size_t)b->n_frames;
    // per-tick gravity (TVEXPONENTIAL only): evaluated on the host exactly as get_gravity(seconds) does, one pair per tick
    const float *d_gtab = nullptr;
    if(b->frame_seconds != nullptr && t.cfg.tsmoothing == WF_TSMOOTH_TVEXPONENTIAL)
    {
        int rcg = ensure(e, &e->s_gtab, &e->s_gtab_cap, 2 * T);
        if(rcg)
            return rcg;
        e->h_gtab.resize(2 * T);
        for(size_t i = 0; i < T; ++i)
        {
            const float g = gravity_for(t.cfg, b->frame_seconds[i]);
            e->h_gtab[2 * i] = g;
            e->h_gtab[2 * i + 1] = 1.0f - g;
        }
        WF_CUDA(e, cudaMemcpyAsync(e->s_gtab, e->h_gtab.data(), 2 * T * sizeof(float), cudaMemcpyHostToDevice, st));
        d_gtab = e->s_gtab;
    }
    bool dev_ptrs = false;
    {
        // Live ticks (one source, one frame: tens of KB) in page-locked, device-mapped host buffers (wf_host_alloc) skip the
        // staging copies altogether: the kernel reads the frame and writes the spectrum over PCIe itself, so a tick costs one
        // launch + one synchronisation.  Every buffer of the batch must be device-addressable for that.
        const void *ptrs[9] = {b->pcm, b->input_rms, b->skip_mask, b->out_db, b->out_points, b->out_silent, b->out_peak, b->out_pixels,
                               b->out_min};
        const bool small = S * T * (size_t)cc * (size_t)N * sizeof(float) <= (1u << 20);
        if(e->zc_valid && memcmp(ptrs, e->zc_ptrs, sizeof(ptrs)) == 0)
            dev_ptrs = e->zc_dev || (e->zc_ok && small && e->zero_copy); // same buffers as the last call, already classified
        else
        {
            const int kpcm = ptr_kind(b->pcm);
            bool zc = (kpcm == 2); // every buffer device-addressable?
            for(int i = 1; i < 9 && zc; ++i)
                zc = (ptrs[i] == nullptr) || (ptr_kind(ptrs[i]) != 0);
            memcpy(e->zc_ptrs, ptrs, sizeof(ptrs));
            e->zc_dev = (kpcm == 1);
            e->zc_ok = zc;
            e->zc_valid = true;
            dev_ptrs = e->zc_dev || (zc && small && e->zero_copy);
        }
    }

    if(dev_ptrs)
    {
        WF_CUDA(e, cudaEventRecord(e->ev0, st));
        if(b->out_peak)
        {
            int rc = fill_device(e, b->out_peak, (long long)T, -INFINITY, st);
            if(rc)
                return rc;
        }
        int rc = launch_range(e, b, st, 0, b->n_streams, b->pcm, b->input_rms, b->skip_mask, b->out_db, b->out_points,
                              b->out_silent, b->out_peak, b->out_pixels, b->out_min, d_gtab);
        if(rc)
            return rc;
        WF_CUDA(e, cudaEventRecord(e->ev1, st));
        e->ev_valid = true;
        return WF_OK;
    }

    // ---- host buffers: stage through device memory, chunked over streams so that the H2D copy of chunk i+1, the
    //      kernel of chunk i and the D2H copy of chunk i-1 overlap (PCIe is full duplex; pinned memory required for
    //      real overlap, pageable memory still works but serialises) ----
    const size_t per_stream_span = (size_t)(cc - 1) * (size_t)b->channel_stride + (T - 1) * (size_t)b->hop + (size_t)N;
    const size_t span = (S - 1) * (size_t)b->stream_stride + per_stream_span;
    int rc;
    if((rc = ensure(e, &e->s_pcm, &e->s_pcm_cap, span)))
        return rc;
    float *d_out_db = nullptr, *d_out_points = nullptr, *d_rms = nullptr, *d_peak = nullptr;
    unsigned char *d_skip = nullptr, *d_silent = nullptr;
    if(b->out_db)
    {
        if((rc = ensure(e, &e->s_out_db, &e->s_out_db_cap, S * T * dch * B)))
            return rc;
        d_out_db = e->s_out_db;
    }
    if(b->out_points)
    {
        if((rc = ensure(e, &e->s_out_points, &e->s_out_points_cap, S * T * dch * t.num_points)))
            return rc;
        d_out_points = e->s_out_points;
    }
    if(b->input_rms)
    {
        if((rc = ensure(e, &e->s_rms, &e->s_rms_cap, S * T)))
            return rc;
        d_rms = e->s_rms;
    }
    if(b->skip_mask)
    {
        if((rc = ensure(e, &e->s_skip, &e->s_skip_cap, S * T)))
            return rc;
        d_skip = e->s_skip;
    }
    if(b->out_silent)
    {
        if((rc = ensure(e, &e->s_silent, &e->s_silent_cap, S * T)))
            return rc;
        d_silent = e->s_silent;
    }
    if(b->out_peak)
    {
        if((rc = ensure(e, &e->s_peak, &e->s_peak_cap, T)))
            return rc;
        d_peak = e->s_peak;
    }
    float *d_px = nullptr, *d_min = nullptr;
    if(b->out_pixels)
    {
        if((rc = ensure(e, &e->s_px, &e->s_px_cap, S * T * dch * t.num_points)))
            return rc;
        d_px = e->s_px;
    }
    if(b->out_min)
    {
        if((rc = ensure(e, &e->s_min, &e->s_min_cap, S * T * 2)))
            return rc;
        d_min = e->s_min;
    }
    if(!e->s_h2d)
    {
        WF_CUDA(e, cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking));
        WF_CUDA(e, cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking));
        for(auto &ev : e->chunk_in)
            WF_CUDA(e, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        for(auto &ev : e->chunk_k)
            WF_CUDA(e, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        WF_CUDA(e, cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
        WF_CUDA(e, cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming));
    }
    const size_t in_bytes = span * sizeof(float);
    int nchunks = (int)std::min<size_t>(std::min<size_t>(wf_engine::kMaxChunks, S), std::max<size_t>(1, in_bytes >> 25));
    const int per = (int)((S + nchunks - 1) / nchunks);
    nchunks = (int)((S + per - 1) / per);

    WF_CUDA(e, cudaEventRecord(e->ev0, st));
    WF_CUDA(e, cudaEventRecord(e->ev_fork, st));
    WF_CUDA(e, cudaStreamWaitEvent(e->s_h2d, e->ev_fork, 0));
    WF_CUDA(e, cudaStreamWaitEvent(e->s_d2h, e->ev_fork, 0));
    if(d_peak)
    {
        if((rc = fill_device(e, d_peak, (long long)T, -INFINITY, st)))
            return rc;
    }
    for(int c = 0; c < nchunks; ++c)
    {
        const int s0 = c * per;
        const int cnt = std::min<int>(per, (int)S - s0);
        const size_t off = (size_t)s0 * (size_t)b->stream_stride;
        const size_t cspan = (size_t)(cnt - 1) * (size_t)b->stream_stride + per_stream_span;
        WF_CUDA(e, cudaMemcpyAsync(e->s_pcm + off, b->pcm + off, cspan * sizeof(float), cudaMemcpyHostToDevice, e->s_h2d));
        if(d_rms)
            WF_CUDA(e, cudaMemcpyAsync(d_rms + (size_t)s0 * T, b->input_rms + (size_t)s0 * T, (size_t)cnt * T * sizeof(float),
                                       cudaMemcpyHostToDevice, e->s_h2d));
        if(d_skip)
            WF_CUDA(e, cudaMemcpyAsync(d_skip + (size_t)s0 * T, b->skip_mask + (size_t)s0 * T, (size_t)cnt * T,
                                       cudaMemcpyHostToDevice, e->s_h2d));
        WF_CUDA(e, cudaEventRecord(e->chunk_in[c], e->s_h2d));
        WF_CUDA(e, cudaStreamWaitEvent(st, e->chunk_in[c], 0));
        if((rc = launch_range(e, b, st, s0, cnt, e->s_pcm, d_rms, d_skip, d_out_db, d_out_points, d_silent, d_peak, d_px,
                              d_min, d_gtab)))
            return rc;
        WF_CUDA(e, cudaEventRecord(e->chunk_k[c], st));
        WF_CUDA(e, cudaStreamWaitEvent(e->s_d2h, e->chunk_k[c], 0));
        if(b->out_db)
            WF_CUDA(e, cudaMemcpyAsync(b->out_db + (size_t)s0 * T * dch * B, d_out_db + (size_t)s0 * T * dch * B,
                                       (size_t)cnt * T * dch * B * sizeof(float), cudaMemcpyDeviceToHost, e->s_d2h));
        if(b->out_points)
            WF_CUDA(e, cudaMemcpyAsync(b->out_points + (size_t)s0 * T * dch * t.num_points,
                                       d_out_points + (size_t)s0 * T * dch * t.num_points,
                                       (size_t)cnt * T * dch * t.num_points * sizeof(float), cudaMemcpyDeviceToHost, e->s_d2h));
        if(b->out_silent)
            WF_CUDA(e, cudaMemcpyAsync(b->out_silent + (size_t)s0 * T, d_silent + (size_t)s0 * T, (size_t)cnt * T,
                                       cudaMemcpyDeviceToHost, e->s_d2h));
        if(b->out_pixels)
            WF_CUDA(e, cudaMemcpyAsync(b->out_pixels + (size_t)s0 * T * dch * t.num_points,
                                       d_px + (size_t)s0 * T * dch * t.num_points,
                                       (size_t)cnt * T * dch * t.num_points * sizeof(float), cudaMemcpyDeviceToHost, e->s_d2h));
        if(b->out_min)
            WF_CUDA(e, cudaMemcpyAsync(b->out_min + (size_t)s0 * T * 2, d_min + (size_t)s0 * T * 2,
                                       (size_t)cnt * T * 2 * sizeof(float), cudaMemcpyDeviceToHost, e->s_d2h));
    }
    WF_CUDA(e, cudaEventRecord(e->ev1, st));
    e->ev_valid = true;
    if(b->out_peak) // complete only after the last chunk's kernel
        WF_CUDA(e, cudaMemcpyAsync(b->out_peak, d_peak, T * sizeof(float), cudaMemcpyDeviceToHost, e->s_d2h));
    WF_CUDA(e, cudaEventRecord(e->ev_join, e->s_d2h));
    WF_CUDA(e, cudaStreamWaitEvent(st, e->ev_join, 0)); // the caller's stream completes when the results are home
    return WF_OK;
}

int wf_process(wf_engine *e, const wf_batch *b)
{
    int rc = wf_process_async(e, b, nullptr);
    if(rc)
        return rc;
    WF_CUDA(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

int wf_synchronize(wf_engine *e)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    WF_CUDA(e, cudaSetDevice(e->device));
    WF_CUDA(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

int wf_reset_state(wf_engine *e, int32_t first, int32_t count)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    if(first < 0 || count < 0 || (int64_t)first + count > e->tab.cfg.max_streams)
        return set_err(e, WF_ERR_CAPACITY, "reset range out of bounds");
    if(count == 0)
        return WF_OK;
    WF_CUDA(e, cudaSetDevice(e->device));
    // on the device, per stream, so that a stream that is already silent keeps its buffers exactly as the reference's
    // early return does (src/source_generic.cpp:38-39)
    const Tables &t = e->tab;
    const bool below = !(t.db_min > (float)(t.cfg.floor_db - 10));
    const unsigned char fl = (unsigned char)(1u | (below ? 6u : 0u));
    const size_t B = (size_t)t.B;
    spectrum_reset_kernel<<<std::min(count, e->sm_count * 8), 256, 0, e->stream>>>(
        e->d_state + (size_t)first * t.cfg.capture_channels * B, e->d_hold + (size_t)first * t.output_channels * B, e->d_flags + first,
        count, (int)(t.cfg.capture_channels * B), (int)(t.output_channels * B), (int)(t.display_channels * B), t.db_min, fl);
    WF_CUDA(e, cudaGetLastError());
    e->launches++;
    WF_CUDA(e, cudaStreamSynchronize(e->stream));
    return WF_OK;
}

int wf_get_state(wf_engine *e, int32_t first, int32_t count, float *tsmooth, float *hold_db, uint8_t *flags)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    const Tables &t = e->tab;
    if(first < 0 || count < 0 || (int64_t)first + count > t.cfg.max_streams)
        return set_err(e, WF_ERR_CAPACITY, "state range out of bounds");
    WF_CUDA(e, cudaSetDevice(e->device));
    {
        const int rc = materialize_hold(e, e->stream);
        if(rc)
            return rc;
    }
    WF_CUDA(e, cudaStreamSynchronize(e->stream));
    const size_t cc = (size_t)t.cfg.capture_channels, och = (size_t)t.output_channels, B = (size_t)t.B;
    if(tsmooth)
        WF_CUDA(e, cudaMemcpy(tsmooth, e->d_state + first * cc * B, count * cc * B * sizeof(float), cudaMemcpyDeviceToHost));
    if(hold_db)
        WF_CUDA(e, cudaMemcpy(hold_db, e->d_hold + first * och * B, count * och * B * sizeof(float), cudaMemcpyDeviceToHost));
    if(flags)
    {
        WF_CUDA(e, cudaMemcpy(flags, e->d_flags + first, (size_t)count, cudaMemcpyDeviceToHost));
        for(int i = 0; i < count; ++i)
            flags[i] &= 1u;
    }
    return WF_OK;
}

int wf_set_state(wf_engine *e, int32_t first, int32_t count, const float *tsmooth, const float *hold_db,
                 const uint8_t *flags)
{
    if(!e)
        return WF_ERR_INVALID_ARG;
    const Tables &t = e->tab;
    if(first < 0 || count < 0 || (int64_t)first + count > t.cfg.max_streams)
        return set_err(e, WF_ERR_CAPACITY, "state range out of bounds");
    WF_CUDA(e, cudaSetDevice(e->device));
    {
        const int rc = materialize_hold(e, e->stream);
        if(rc)
            return rc;
    }
    WF_CUDA(e, cudaStreamSynchronize(e->stream));
    const size_t cc = (size_t)t.cfg.capture_channels, och = (size_t)t.output_channels, B = (size_t)t.B;
    if(tsmooth)
        WF_CUDA(e, cudaMemcpy(e->d_state + first * cc * B, tsmooth, count * cc * B * sizeof(float), cudaMemcpyHostToDevice));
    std::vector<unsigned char> fl((size_t)count);
    WF_CUDA(e, cudaMemcpy(fl.data(), e->d_flags + first, (size_t)count, cudaMemcpyDeviceToHost));
    if(hold_db)
    {
        WF_CUDA(e, cudaMemcpy(e->d_hold + first * och * B, hold_db, count * och * B * sizeof(float), cudaMemcpyHostToDevice));
        const float thr = (float)(t.cfg.floor_db - 10);
        for(int s = 0; s < count; ++s)
        {
            unsigned char bits = 0;
            for(int d = 0; d < t.display_channels; ++d)
            {
                bool all_below = true;
                const float *row = hold_db + ((size_t)s * och + d) * B;
                for(size_t k = 0; k < B; ++k)
                    if(row[k] > thr)
                    {
                        all_below = false;
                        break;
                    }
                if(all_below)
                    bits |= (unsigned char)(2u << d);
            }
            if(t.display_channels == 1)
                bits |= 4u;
            fl[s] = (unsigned char)((fl[s] & 1u) | bits);
        }
    }
    if(flags)
        for(int s = 0; s < count; ++s)
            fl[s] = (unsigned char)((fl[s] & ~1u) | (flags[s] & 1u));
    WF_CUDA(e, cudaMemcpy(e->d_flags + first, fl.data(), (size_t)count, cudaMemcpyHostToDevice));
    return WF_OK;
}

int wf_peak_normalize(wf_engine *e, float *data, int32_t n_streams, int32_t n_frames, int32_t row_len,
                      const float *peak, float target_db, float max_gain, void *cuda_stream)
{
    if(!e || !data || !peak || n_streams < 0 || n_frames < 0 || row_len < 1)
        return e ? set_err(e, WF_ERR_INVALID_ARG, "bad peak_normalize arguments") : WF_ERR_INVALID_ARG;
    NvtxRange nvtx("wf_peak_normalize");
    if(n_streams == 0 || n_frames == 0)
        return WF_OK;
    WF_CUDA(e, cudaSetDevice(e->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : e->stream;
    const int rows_per_frame = e->tab.display_channels;
    const size_t total = (size_t)n_streams * n_frames * rows_per_frame * row_len;
    const bool dev = is_device_ptr(data);
    float *d_data = data;
    const float *d_peak = peak;
    if(!dev)
    {
        int rc;
        if((rc = ensure(e, &e->s_out_db, &e->s_out_db_cap, total)))
            return rc;
        if((rc = ensure(e, &e->s_peak, &e->s_peak_cap, (size_t)n_frames)))
            return rc;
        WF_CUDA(e, cudaMemcpyAsync(e->s_out_db, data, total * sizeof(float), cudaMemcpyHostToDevice, st));
        WF_CUDA(e, cudaMemcpyAsync(e->s_peak, peak, (size_t)n_frames * sizeof(float), cudaMemcpyHostToDevice, st));
        d_data = e->s_out_db;
        d_peak = e->s_peak;
    }
    else if(!is_device_ptr(peak))
    {
        int rc;
        if((rc = ensure(e, &e->s_peak, &e->s_peak_cap, (size_t)n_frames)))
            return rc;
        WF_CUDA(e, cudaMemcpyAsync(e->s_peak, peak, (size_t)n_frames * sizeof(float), cudaMemcpyHostToDevice, st));
        d_peak = e->s_peak;
    }
    WF_CUDA(e, cudaEventRecord(e->ev0, st));
    const long long rows = (long long)n_streams * n_frames * rows_per_frame;
    const int grid = (int)std::min<long long>(rows, (long long)e->sm_count * 16);
    peak_normalize_kernel<<<grid, 256, 0, st>>>(d_data, n_streams, n_frames, rows_per_frame, row_len, d_peak, target_db,
                                                max_gain);
    WF_CUDA(e, cudaGetLastError());
    e->launches++;
    WF_CUDA(e, cudaEventRecord(e->ev1, st));
    e->ev_valid = true;
    if(!dev)
    {
        WF_CUDA(e, cudaMemcpyAsync(data, d_data, total * sizeof(float), cudaMemcpyDeviceToHost, st));
        WF_CUDA(e, cudaStreamSynchronize(st));
    }
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

float wf_last_kernel_ms(wf_engine *e)
{
    if(!e || !e->ev_valid)
        return -1.0f;
    if(cudaEventSynchronize(e->ev1) != cudaSuccess)
        return -1.0f;
    float ms = -1.0f;
    if(cudaEventElapsedTime(&ms, e->ev0, e->ev1) != cudaSuccess)
        return -1.0f;
    return ms;
}

} // extern "C"
