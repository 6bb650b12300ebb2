// wf_kparams.hpp — the parameter block every spectrum kernel takes (KParams), and the display-table size that routing and
// the kernels both need.  No device code: the engine's host file includes it without compiling any kernel.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace wf {

struct KParams {
    // input
    const float *pcm;                // float or int16_t samples (the kernel's sample type, see wf_pcm.cuh)
    long long stream_stride, channel_stride;
    int n_streams, n_frames, hop;
    int aligned8; // every frame start is 8-byte aligned -> sample-pair loads
    const float *input_rms;          // [n_streams][n_frames] or null
    const unsigned char *skip_mask;  // [n_streams][n_frames] or null
    // tables
    const float2 *window2; // window as float2[N/2] or null
    const float *window;   // same table, scalar view
    const float2 *tw;      // W_M^k
    const float2 *tw_post; // W_N^k, k < M
    const float *slope;    // or null
    const float *rolloff;  // or null
    // per-stream persistent state (already offset by first_stream)
    float *state;          // [streams][CC][B]   m_tsmooth_buf / last linear magnitude
    float *hold_db;        // [streams][OCH][B]  m_decibels as left by the last tick
    unsigned char *flags;  // [streams] bit0 last_silent, bit1/2 prev outputs of display slot 0/1 all <= floor-10
    // outputs
    float *out_db;             // [streams][frames][DCH][B] or null
    float *out_points;         // [streams][frames][DCH][n_points] or null
    unsigned char *out_silent; // [streams][frames] or null
    float *out_peak;           // [frames] or null (atomic max)
    // scalars
    float coef_half;  // (2 / window_sum) / 2
    float g, g2;      // gravity, 1 - gravity
    const float2 *g_tab; // optional [n_frames] (g, 1-g) per tick: TV-exponential smoothing with per-tick frame times
    int tsmooth;      // != 0: EMA enabled
    int fast_peaks;
    int stereo, och, dch;
    int gate;
    float floor_m10;  // (float)(floor - 10)
    float db_min;
    int normalize;
    float vol_target, max_gain;
    int write_hold;   // write final m_decibels mirror to hold_db at the end of the call
    int lazy_hold;    // N=2048 warp-per-stream kernel: leave the mirror implicit (flags bit 3) when it equals dbfs(state)
    int disp_bytes;   // warp-per-stream kernels with display outputs: extra shared memory per warp (dB row + display scratch)
    int disp_tab_bytes; // ... and per CTA (the display stage's setup tables)
    int split;        // N=2048 warp-per-stream kernel: cut an SM's frames into equal runs per warp (streams may change warps mid-call)
    // interpolation
    const float *interp_idx;
    const float *interp_w;
    const int *band_widths;
    const int *band_offsets;
    int n_points, taps, radius, display_bar, interp_mode;
    int n_sample;   // bars with a Lanczos / Catmull-Rom kernel: sample points of all bands (sum of band_widths), else 0
    int scratch_q;  // display scratch per stream = 4 * scratch_q floats (>= 4*n_points + dch*n_sample)
    const float *gauss_w;
    int gauss_radius, gauss_size;
    float gauss_sum;
    int filter;
    // display stage (dB -> pixels)
    float *out_pixels;     // [streams][frames][DCH][n_points] or null
    float *out_min;        // [streams][frames][2] or null
    float px_lo, px_hi;    // lerp endpoints: (0, cpos - channel_offset) for the curve, (border_top, border_bottom) for bars
    float px_cpos;         // initial miny
    float ceiling_f;       // (float)m_ceiling
    float dbrange_f;       // (float)(m_ceiling - m_floor)
    int mirror;
};

// floats of shared memory the display stage's setup tables take when a kernel stages them (stage_display_tables,
// wf_kernels.cuh): weights padded to 16 bytes first, then indices, Gaussian, band widths, band offsets
__host__ __device__ inline size_t display_table_floats(const KParams &p)
{
    const size_t n_idx = (p.n_sample > 0) ? (size_t)p.n_sample : (size_t)p.n_points;
    const size_t n_w = (p.interp_mode != 0) ? n_idx * (size_t)p.taps : 0;
    return ((n_w + 3) & ~(size_t)3) + n_idx + (p.filter ? (size_t)p.gauss_size : 0) + (p.display_bar ? 2 * (size_t)p.n_points : 0);
}

} // namespace wf
