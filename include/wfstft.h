/* wfstft.h — C ABI of libwfstft.so, the H100 (sm_90a) batched STFT engine that drops in behind
 * phandasm/waveform's spectrum backend seam.
 *
 * What it replaces (paths relative to the reference tree):
 *   - the pure virtual  WAVSource::tick_spectrum(float)            src/source.hpp:275
 *     and its three CPU implementations                            src/source_generic.cpp:26-180,
 *                                                                  src/source_avx.cpp:29-200, src/source_avx2.cpp:24-209
 *   - the only FFTW calls the plugin makes                         src/source.cpp:1187 (plan), src/source_generic.cpp:106
 *                                                                  (execute), src/source.cpp:803 (destroy)
 *   - table construction done in WAVSource::update                 src/source.cpp:1190-1234 (window), :1282-1290 (slope),
 *                                                                  :898-918 (roll-off), :837-896 (interpolation)
 *   - the render-time interpolation / smoothing of m_decibels      src/source.cpp:1381-1406, :1510-1546,
 *                                                                  src/filter.hpp:133-211, src/filter_fma3.cpp:23-219
 *
 * Conventions
 *   - plain C, no exceptions; every function returns WF_OK (0) or a negative wf_status;
 *     wf_last_error() gives a human-readable reason for the last failure on that engine.
 *   - one engine handle is externally serialised (the plugin holds m_mtx around tick/render/update,
 *     src/source.cpp:1326,1348,1079); different handles may be used concurrently from different threads.
 *   - data pointers in a wf_batch may be HOST or DEVICE pointers (all of one kind per call, detected with
 *     cudaPointerGetAttributes).  Host buffers are copied to / from device staging buffers inside the call, chunked so that
 *     H2D, kernel and D2H overlap — which needs page-locked (pinned) caller buffers; pageable ones work but serialise.
 *     Small batches in device-mapped pinned memory (wf_host_alloc) are processed in place, without copies (live ticks).
 *   - the engine owns all device memory (tables, per-stream EMA state, staging); the caller owns pcm/out.
 *   - there is no CPU fallback: without a CUDA device wf_create fails with WF_ERR_NO_DEVICE.
 */
#ifndef WFSTFT_H
#define WFSTFT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WF_ABI_VERSION 2

typedef enum wf_status {
    WF_OK = 0,
    WF_ERR_INVALID_ARG = -1,
    WF_ERR_UNSUPPORTED_FFT_SIZE = -2, /* never a silent approximation: unsupported N is an error */
    WF_ERR_CUDA = -3,
    WF_ERR_NO_DEVICE = -4,
    WF_ERR_OOM = -5,
    WF_ERR_CAPACITY = -6, /* n_streams > max_streams */
    WF_ERR_ABI = -7
} wf_status;

/* Enumerations mirror src/source.hpp:32-93 (same order). */
typedef enum { WF_WINDOW_NONE, WF_WINDOW_HANN, WF_WINDOW_HAMMING, WF_WINDOW_BLACKMAN, WF_WINDOW_BLACKMAN_HARRIS,
               WF_WINDOW_POWER_OF_SINE } wf_window;          /* FFTWindow */
typedef enum { WF_INTERP_POINT, WF_INTERP_LANCZOS, WF_INTERP_CATROM } wf_interp;          /* InterpMode */
typedef enum { WF_FILTER_NONE, WF_FILTER_GAUSS } wf_filter;                                 /* FilterMode */
typedef enum { WF_TSMOOTH_NONE, WF_TSMOOTH_EXPONENTIAL, WF_TSMOOTH_TVEXPONENTIAL } wf_tsmooth; /* TSmoothingMode */
typedef enum { WF_DISPLAY_CURVE, WF_DISPLAY_BAR } wf_display; /* DisplayMode CURVE / BAR+STEPPED_BAR */

/* DSP-relevant subset of the plugin's settings: what WAVSource::get_settings (src/source.cpp:501-674)
 * leaves in the m_* members that tick_spectrum / init_interp / init_rolloff read.  wf_create applies the
 * same clamps (fft_size >= 128 and &-16, cutoff and floor/ceiling sanity, :562-577). */
typedef struct wf_config {
    uint32_t struct_size;      /* = sizeof(wf_config); ABI check */
    int32_t device;            /* CUDA device ordinal, -1 = current device */
    int32_t max_streams;       /* independent sources whose EMA state the engine keeps (>= 1) */
    uint32_t sample_rate;      /* m_audio_info.samples_per_sec */
    int32_t capture_channels;  /* m_capture_channels: 1 or 2 (src/source.cpp:1089) */
    int32_t fft_size;          /* m_fft_size */
    int32_t window;            /* wf_window, m_window_func */
    int32_t sine_exponent;     /* m_sine_exponent */
    int32_t tsmoothing;        /* wf_tsmooth, m_tsmoothing */
    float gravity;             /* m_gravity */
    int32_t fast_peaks;        /* m_fast_peaks */
    float slope;               /* m_slope */
    float rolloff_q;           /* m_rolloff_q */
    float rolloff_rate;        /* m_rolloff_rate */
    int32_t cutoff_low;        /* m_cutoff_low  (Hz) */
    int32_t cutoff_high;       /* m_cutoff_high (Hz) */
    int32_t floor_db;          /* m_floor */
    int32_t ceiling_db;        /* m_ceiling */
    int32_t stereo;            /* m_stereo (channel_mode == stereo) */
    int32_t normalize_volume;  /* m_normalize_volume */
    float volume_target;       /* m_volume_target */
    float max_gain;            /* m_max_gain */
    int32_t silence_gate;      /* 1 = reference "wait for gravity" gating, src/source_generic.cpp:63-95 */
    int32_t display_mode;      /* wf_display */
    int32_t width;             /* m_width */
    int32_t bar_width;         /* m_bar_width */
    int32_t bar_gap;           /* m_bar_gap */
    int32_t log_scale;         /* m_log_scale */
    int32_t mirror_freq_axis;  /* m_mirror_freq_axis */
    int32_t interp_mode;       /* wf_interp, m_interp_mode */
    int32_t filter_mode;       /* wf_filter, m_filter_mode */
    float filter_radius;       /* m_filter_radius */
    /* display stage (src/source.cpp:1408-1424, 1473-1565): dB -> pixel height of curve points / bars */
    int32_t height;            /* m_height (after the radial adjustment, if any) */
    int32_t channel_spacing;   /* m_channel_spacing (get_settings zeroes it unless stereo, src/source.cpp:579-580) */
    int32_t rounded_caps;      /* m_rounded_caps (bars only) */
    int32_t min_bar_height;    /* m_min_bar_height */
} wf_config;

/* Facts derived at create time. */
typedef struct wf_info {
    int32_t fft_size;         /* after clamping */
    int32_t bins;             /* fft_size / 2 (Nyquist and above discarded, src/source_avx2.cpp:29) */
    int32_t capture_channels;
    int32_t output_channels;  /* m_output_channels, src/source.cpp:1170 */
    int32_t display_channels; /* m_stereo ? 2 : 1 */
    int32_t num_points;       /* display points per channel: width (curve) or num_bars (bars) */
    int32_t num_bars;
    int32_t interp_taps;      /* 8 (Lanczos a=4), 4 (Catmull-Rom) or 0 (point) */
    int32_t n_interp_indices;
    float window_sum;         /* m_window_sum */
    float db_min;             /* DB_MIN = 20*log10f(FLT_MIN), src/source.cpp:43 */
    int32_t device;
    int32_t sm_count;
} wf_info;

typedef enum wf_table {
    WF_TABLE_WINDOW = 0,        /* float[fft_size]   m_window_coefficients */
    WF_TABLE_SLOPE = 1,         /* float[bins]       m_slope_modifiers     */
    WF_TABLE_ROLLOFF = 2,       /* float[bins]       m_rolloff_modifiers   */
    WF_TABLE_INTERP_INDICES = 3,/* float[n_interp_indices] m_interp_indices */
    WF_TABLE_INTERP_WEIGHTS = 4,/* float[n_interp_indices*interp_taps] m_interp_kernel.weights */
    WF_TABLE_BAND_WIDTHS = 5,   /* int32 stored as float-sized words [num_bars] m_band_widths */
    WF_TABLE_GAUSS = 6          /* float[2*ceil(3 sigma)-1] m_kernel.weights */
} wf_table;

/* One call = n_streams independent sources x n_frames consecutive ticks.
 *   frame t of capture channel c of stream s = pcm[s*stream_stride + c*channel_stride + t*hop ... + fft_size)
 * i.e. what CircularBuffer::peek_front hands tick_spectrum on successive ticks (src/source_generic.cpp:55-59)
 * when `hop` new samples arrive per tick.  The EMA recurrence (src/source_generic.cpp:124-132) runs over t
 * inside the call and continues across calls through the engine's per-stream state. */
typedef struct wf_batch {
    uint32_t struct_size;      /* = sizeof(wf_batch) */
    int32_t n_streams;
    int32_t n_frames;
    int32_t hop;               /* samples between consecutive frames (>= 1) */
    int32_t first_stream;      /* state slot of stream 0 of this batch (0 <= first_stream, first+n <= max_streams) */
    float seconds;             /* tick delta for TVEXPONENTIAL gravity (src/source.hpp:301-312); ignored otherwise */
    const float *pcm;          /* planar float PCM, host or device */
    int64_t stream_stride;     /* in floats */
    int64_t channel_stride;    /* in floats */
    const float *input_rms;    /* [n_streams][n_frames] m_input_rms per tick; REQUIRED when normalize_volume is set (else
                                  WF_ERR_INVALID_ARG: never a silent max_gain), ignored otherwise */
    const uint8_t *skip_mask;  /* optional [n_streams][n_frames]: nonzero = "not enough audio" for that tick */
    float *out_db;             /* optional [n_streams][n_frames][display_channels][bins]       m_decibels      */
    float *out_points;         /* optional [n_streams][n_frames][display_channels][num_points] interpolated dB */
    uint8_t *out_silent;       /* optional [n_streams][n_frames] m_last_silent after the tick */
    float *out_peak;           /* optional [n_frames]: max over streams/channels/bins>=1 of the dB output
                                  (input to the cross-channel peak normalisation; all-reduce(max) it across GPUs) */
    float *out_pixels;         /* optional [n_streams][n_frames][display_channels][num_points]: what render_curve /
                                  render_bars leave in m_interp_bufs — pixel heights after lerp/clamp and mirroring */
    float *out_min;            /* optional [n_streams][n_frames][2]: (miny, minpos) of the tick (pulse colouring) */
    const float *frame_seconds; /* optional HOST array [n_frames]: the `seconds` argument of each tick (src/source.cpp:1324).
                                  Only TVEXPONENTIAL smoothing looks at it: gravity = exp(-seconds / (gravity * 0.1934...))
                                  is then evaluated per tick as get_gravity() does (src/source.hpp:301-312), so a batch
                                  recorded with jittering frame times replays exactly.  NULL: `seconds` for every tick. */
} wf_batch;

typedef struct wf_engine wf_engine;

int wf_abi_version(void);
const char *wf_strerror(int status);
const char *wf_last_error(const wf_engine *e);

/* Fill cfg with the plugin's defaults (src/source.cpp:119-174); sets struct_size. */
void wf_config_init(wf_config *cfg);

/* ≙ callbacks::create + WAVSource::update (src/source.cpp:87-102, 1077-1322): validates settings, builds all
 * tables, allocates device state.  Unsupported fft_size -> WF_ERR_UNSUPPORTED_FFT_SIZE. */
int wf_create(const wf_config *cfg, wf_engine **out);
/* ≙ WAVSource::~WAVSource / free_bufs (src/source.cpp:782-808). */
void wf_destroy(wf_engine *e);

int wf_get_info(const wf_engine *e, wf_info *info);
/* Copies a host copy of a table; returns element count (>= 0) or a negative status. out may be NULL. */
int64_t wf_get_table(const wf_engine *e, int which, float *out, int64_t capacity);
/* ≙ WAVSource::get_gravity(seconds), src/source.hpp:301-312. */
float wf_gravity(const wf_engine *e, float seconds);

/* The same setup-time tables, computed from a config WITHOUT creating an engine (no device needed): lets a host
 * (or a CPU-only test) check them against the plugin's own m_* tables.  Returns element count or a negative status;
 * info (optional) receives the derived facts (device/sm_count = -1). */
int64_t wf_preview_table(const wf_config *cfg, int which, float *out, int64_t capacity, wf_info *info);

/* ≙ tick_spectrum for every (stream, tick) of the batch (+ render-time interpolation when out_points is set).
 * Blocking: returns after results are in the caller's buffers. */
int wf_process(wf_engine *e, const wf_batch *batch);
/* Same, enqueued on `cuda_stream` (a cudaStream_t; NULL = the engine's own stream) without synchronising.
 * With host pointers the copies are enqueued on the same stream (pinned memory recommended). */
int wf_process_async(wf_engine *e, const wf_batch *batch, void *cuda_stream);
int wf_synchronize(wf_engine *e);

/* ≙ the timeout / hidden branch (src/source_generic.cpp:36-48): zero EMA state, outputs := DB_MIN,
 * m_last_silent := true for streams [first, first+count). */
int wf_reset_state(wf_engine *e, int32_t first_stream, int32_t count);

/* Checkpoint / restore of the per-stream recurrence state (host buffers):
 *   tsmooth  [count][capture_channels][bins]   m_tsmooth_buf
 *   hold_db  [count][output_channels][bins]    m_decibels as left by the last tick
 *   flags    [count]                           bit0 = m_last_silent */
int wf_get_state(wf_engine *e, int32_t first_stream, int32_t count, float *tsmooth, float *hold_db, uint8_t *flags);
int wf_set_state(wf_engine *e, int32_t first_stream, int32_t count, const float *tsmooth, const float *hold_db,
                 const uint8_t *flags);

/* Cross-channel peak normalisation (BASELINE config 5; generalises the single-source volume normalisation of
 * src/source_generic.cpp:161-167 to a peak shared by all channels on all GPUs):
 *   gain[t] = min(target_db - peak[t], max_gain);  out[s][t][ch][k] += gain[t]  for k >= 1
 * `peak` is the (all-reduced) wf_batch.out_peak array; `data` is an out_db-shaped ([..][bins]) or
 * out_points-shaped ([..][num_points]) buffer, `row_len` its innermost length.  Device or host pointers. */
int wf_peak_normalize(wf_engine *e, float *data, int32_t n_streams, int32_t n_frames, int32_t row_len,
                      const float *peak, float target_db, float max_gain, void *cuda_stream);

/* Page-locked, device-mapped host memory for the live path (≙ the plugin's AlignedBuffer for m_fft_input / m_decibels,
 * src/aligned_buffer.hpp:30-80, but visible to the GPU).  When EVERY buffer of a small batch (at most 1 MiB of PCM) lives in
 * memory from wf_host_alloc (or on the device), wf_process* launches the kernel directly on those buffers — no staging
 * copies: one launch + one synchronisation per tick.  Pageable host buffers keep working (staged, chunked, overlapped).
 * Returns NULL on failure; wf_host_free(NULL) is a no-op. */
void *wf_host_alloc(size_t bytes);
void wf_host_free(void *p);

/* Number of kernel launches this engine has issued (bench.py reports it as gpu_launches). */
int64_t wf_launch_count(const wf_engine *e);
/* Name (template arguments and launch geometry included) of the spectrum kernel the most recent wf_process* call
 * dispatched to, e.g. "stft2048_fast_kernel<16,1,1,0> grid 132 x 16 warps"; "" before the first call.  Valid until the
 * next call on this engine.  bench.py reports it as roofline.kernel, the tests assert the routing with it. */
const char *wf_last_kernel_name(const wf_engine *e);
/* Device time (ms) of the kernel section of the most recent wf_process / wf_process_async / wf_peak_normalize call,
 * measured with CUDA events on the launching stream; < 0 if none. Synchronises on the recorded events. */
float wf_last_kernel_ms(wf_engine *e);


/* ---------------------------------------------------------------------------------------------------------------
 * Level meter and RMS feed — the other reductions behind the same backend seam (SURVEY.md §8(f) rank 4, §8(a) a9):
 *   WAVSource::tick_meter            src/source.hpp:276, src/source_generic.cpp:182-270, src/source_avx.cpp:202-301
 *   WAVSource::update_input_rms      src/source.hpp:277, src/source_generic.cpp:392-403, src/source_avx.cpp:303-322
 *   the ring that feeds it           src/source.cpp:810-836 (sync_rms_buffer), :1842-1871 (capture_audio)
 *   meter setup                      src/source.cpp:1105-1128
 * A wf_meter keeps, per stream, the ring of the last `window` samples (m_decibels repurposed, :205-222), the EMA value
 * m_meter_buf and m_last_silent.  One call = n_streams sources x n_ticks ticks; tick t consumes samples
 * [t*hop, (t+1)*hop) of each capture channel (everything captured since the previous tick).
 * Peak values are bit-exact; RMS values are summed in blocks (not in ring order) and agree to ~1e-6 relative. */
typedef enum { WF_METER_PEAK = 0, WF_METER_RMS = 1, WF_METER_INPUT_RMS = 2 } wf_meter_mode;

typedef struct wf_meter_config {
    uint32_t struct_size;     /* = sizeof(wf_meter_config) */
    int32_t device;           /* CUDA device ordinal, -1 = current */
    int32_t max_streams;
    uint32_t sample_rate;     /* m_audio_info.samples_per_sec */
    int32_t capture_channels; /* 1 or 2 */
    int32_t mode;             /* wf_meter_mode: PEAK / RMS = m_meter_rms false / true; INPUT_RMS = the volume-normalisation
                                 feed: sqrt(mean over the last (sample_rate & -16) samples of (max over channels |x|)^2) */
    int32_t meter_ms;         /* m_meter_ms: window = (sample_rate * meter_ms / 1000) & -16 (ignored for INPUT_RMS) */
    int32_t tsmoothing;       /* wf_tsmooth */
    float gravity;            /* m_gravity */
    int32_t fast_peaks;       /* m_fast_peaks */
    int32_t floor_db;         /* m_floor: a channel below floor-10 dB counts as silent */
} wf_meter_config;

typedef struct wf_meter_batch {
    uint32_t struct_size;     /* = sizeof(wf_meter_batch) */
    int32_t n_streams;
    int32_t n_ticks;
    int32_t hop;              /* new samples per tick (>= 1) */
    int32_t first_stream;
    float seconds;            /* tick delta for TVEXPONENTIAL gravity */
    const float *pcm;         /* planar float PCM, host or device: sample i of channel c of stream s at
                                 pcm[s*stream_stride + c*channel_stride + i], i < n_ticks*hop */
    int64_t stream_stride;
    int64_t channel_stride;
    float *out_db;            /* optional [n_streams][n_ticks][capture_channels] m_meter_val (dBFS); unused for INPUT_RMS */
    float *out_lin;           /* optional [n_streams][n_ticks][capture_channels] m_meter_buf;
                                 INPUT_RMS: [n_streams][n_ticks] m_input_rms (feed it to wf_batch.input_rms) */
    uint8_t *out_silent;      /* optional [n_streams][n_ticks] m_last_silent after the tick; unused for INPUT_RMS */
} wf_meter_batch;

typedef struct wf_meter wf_meter;

void wf_meter_config_init(wf_meter_config *cfg); /* plugin defaults: 150 ms, RMS, EMA 0.65, floor -65 (src/source.cpp:119-174) */
int wf_meter_create(const wf_meter_config *cfg, wf_meter **out); /* ≙ WAVSource::update in meter mode */
void wf_meter_destroy(wf_meter *m);
const char *wf_meter_last_error(const wf_meter *m);
int32_t wf_meter_window(const wf_meter *m); /* ring length in samples (m_fft_size in meter mode / m_input_rms_size) */
int wf_meter_process(wf_meter *m, const wf_meter_batch *batch);
int wf_meter_process_async(wf_meter *m, const wf_meter_batch *batch, void *cuda_stream);
/* ≙ the capture-timeout branch of tick_meter (src/source_generic.cpp:184-199): unless already silent, zero the ring,
 * m_meter_buf := 0, m_meter_val := DB_MIN, m_last_silent := true. */
int wf_meter_reset(wf_meter *m, int32_t first_stream, int32_t count);
int64_t wf_meter_launch_count(const wf_meter *m);
float wf_meter_last_kernel_ms(wf_meter *m);

/* ---------------------------------------------------------------------------------------------------------------
 * Waveform (oscilloscope) mode — the third tick_* virtual behind the backend seam (SURVEY.md §8(f) rank 4):
 *   WAVSource::tick_waveform          src/source.hpp:277, src/source_generic.cpp:272-390
 *   its setup                         src/source.cpp:1129-1143 (m_fft_size := m_width, m_waveform_samples, m_waveform_ts := 0),
 *                                     :1243-1248 (start-up zeros in the capture ring), :1181 (m_decibels := DB_MIN)
 * A wf_wave keeps, per stream, the scrolling buffer m_decibels[2][width] and m_last_silent, and per ENGINE the clock the
 * reference derives from packet timestamps (m_audio_ts, m_waveform_ts).  One call = n_streams sources x n_ticks ticks; tick t
 * is preceded by a capture packet of samples [t*hop, (t+1)*hop) of each channel whose end is stamped "now" (get_audio_sync
 * == 0).  Every stream of the engine ticks in every call (the timing state is shared).  The nearest-sample resampling is
 * integer arithmetic on nanosecond timestamps (bit-exact); the dBFS conversion uses log10f (last-bit differences). */
typedef struct wf_wave_config {
    uint32_t struct_size;     /* = sizeof(wf_wave_config) */
    int32_t device;           /* CUDA device ordinal, -1 = current */
    int32_t max_streams;
    uint32_t sample_rate;
    int32_t capture_channels; /* 1 or 2 */
    int32_t stereo;           /* m_stereo */
    int32_t width;            /* m_width: points of the scrolling buffer */
    int32_t meter_ms;         /* m_meter_ms: time span shown */
    int32_t normalize_volume; /* m_normalize_volume */
    float volume_target;      /* m_volume_target */
    float max_gain;           /* m_max_gain */
} wf_wave_config;

typedef struct wf_wave_batch {
    uint32_t struct_size;     /* = sizeof(wf_wave_batch) */
    int32_t n_streams;        /* must equal max_streams */
    int32_t n_ticks;
    int32_t hop;              /* samples per capture packet / tick (>= 1) */
    const float *pcm;         /* planar float PCM, host or device; >= n_ticks*hop samples per channel */
    int64_t stream_stride;
    int64_t channel_stride;
    const float *input_rms;   /* optional [n_streams][n_ticks] m_input_rms per tick (volume normalisation) */
    float *out;               /* [n_streams][n_ticks][display_channels][width] m_decibels after the tick (oldest point first) */
    uint8_t *out_silent;      /* optional [n_streams][n_ticks] m_last_silent after the tick */
} wf_wave_batch;

typedef struct wf_wave wf_wave;

void wf_wave_config_init(wf_wave_config *cfg); /* plugin defaults: width 800, 150 ms (src/source.cpp:119-174) */
int wf_wave_create(const wf_wave_config *cfg, wf_wave **out); /* ≙ WAVSource::update in waveform mode */
void wf_wave_destroy(wf_wave *w);
const char *wf_wave_last_error(const wf_wave *w);
int wf_wave_process(wf_wave *w, const wf_wave_batch *batch);
int wf_wave_process_async(wf_wave *w, const wf_wave_batch *batch, void *cuda_stream);
/* ≙ the hidden / capture-timeout branch (src/source_generic.cpp:280-289): unless already silent, buffers := DB_MIN,
 * m_last_silent := true, for every stream. */
int wf_wave_reset(wf_wave *w);
/* The host-side plan of a call made right after wf_wave_create (no device needed; lets a CPU-only test check the integer
 * timestamp walk against the plugin): counts[t] = points emitted by tick t; src (optional, `capacity` entries) = for every
 * point in order the index of the sample it takes in the call's PCM, or -1 for a start-up zero.  Returns the total number of
 * points or a negative status. */
int64_t wf_wave_preview_plan(const wf_wave_config *cfg, int32_t n_ticks, int32_t hop, int32_t *counts, int32_t *src,
                             int64_t capacity);
int64_t wf_wave_launch_count(const wf_wave *w);
float wf_wave_last_kernel_ms(wf_wave *w);

#ifdef __cplusplus
}
#endif
#endif /* WFSTFT_H */
