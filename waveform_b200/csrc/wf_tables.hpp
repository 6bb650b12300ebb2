// wf_tables.hpp — host-side construction of the setup-time tables of the spectrum path.
//
// This is the engine's equivalent of what WAVSource::update() computes once per settings change
// (reference: src/source.cpp:1077-1322).  Setup is host work in the reference and stays host work here;
// the per-frame hot path (the spectrum kernels) only reads these tables from device memory.
//
// All float expressions follow the reference's operation order so that tables are bit-identical on
// glibc (tests/test_tables.py checks that against the compiled reference).  Compiled with
// -ffp-contract=off.
#pragma once
#include <cstdint>
#include <vector>

#include "wfstft.h"

namespace wf {

struct Tables {
    // normalised settings
    wf_config cfg{};
    int N = 0;               // m_fft_size after clamps (src/source.cpp:562-565)
    int B = 0;               // bins = N/2
    int output_channels = 1; // m_output_channels (src/source.cpp:1170)
    int display_channels = 1;
    int num_bars = 0;
    int num_points = 0;
    float window_sum = 1.0f; // m_window_sum
    float db_min = 0.0f;     // DB_MIN (src/source.cpp:43)
    // display stage: lerp endpoints and initial miny of render_curve / render_bars (src/source.cpp:1365-1373,1481-1493)
    float px_lo = 0.0f, px_hi = 0.0f, px_cpos = 0.0f;

    std::vector<float> window;         // m_window_coefficients (empty = none)
    std::vector<float> slope;          // m_slope_modifiers (empty = off)
    std::vector<float> rolloff;        // m_rolloff_modifiers (empty = off)
    std::vector<float> interp_indices; // m_interp_indices
    std::vector<int32_t> band_widths;  // m_band_widths
    std::vector<int32_t> band_offsets; // exclusive prefix sum of band_widths (engine-side helper)
    std::vector<float> interp_weights; // m_interp_kernel.weights
    int interp_radius = 0;
    int interp_taps = 0;
    std::vector<float> gauss;          // m_kernel.weights
    int gauss_radius = 0;
    float gauss_sum = 0.0f;

    // FFT twiddles (double-evaluated, rounded to float; cf. deps/fftw-3.3.11/kernel/trig.c:57-80)
    std::vector<float> tw;      // interleaved re,im of W_M^k, k < M, M = N/2
    std::vector<float> tw_post; // interleaved re,im of W_N^k, k < M
};

// Applies the get_settings clamps and builds every table.  Returns WF_OK or WF_ERR_INVALID_ARG.
int build_tables(const wf_config &cfg, Tables &out, const char **why);

// The display stage of the waveform mode: init_interp for DisplayMode::WAVEFORM (src/source.cpp:842-846: linear axis over
// bins [0, width - 1], no mirroring, settings forced at :1129-1143), the interpolation kernel and Gaussian of the spectrum
// path's builders, and render_curve's geometry (px_lo = 0, px_hi = cpos - channel_offset, px_cpos).  The get_settings clamps
// of the display settings (floor / ceiling, channel spacing, height) land in out.cfg; N = num_points = width.
int build_wave_tables(const wf_wave_config &cfg, Tables &out, const char **why);

float gravity_for(const wf_config &cfg, float seconds); // WAVSource::get_gravity, src/source.hpp:301-312
float std_lerp(float a, float b, float t);              // std::lerp as libstdc++ evaluates it

} // namespace wf
