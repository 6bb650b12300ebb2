// wf_tables.cpp — see wf_tables.hpp.  Host-only, setup-time.
#include "wf_tables.hpp"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <limits>
#include <numbers>

namespace wf {

namespace {

constexpr float kPi = std::numbers::pi_v<float>;

// a * (b/a)^t: geometric interpolation between a and b (≙ log_interp, src/math_funcs.hpp:25-29)
inline float geo_lerp(float a, float b, float t) { return a * std::pow(b / a, t); }

// ---- FFT window ------------------------------------------------------------------------------------------------
// Every cosine-sum window of the plugin (src/source.cpp:1190-1234) is  w[i] = a0 -+ a1 cos(1*phi) +- a2 cos(2*phi) ...
// with phi = 2 pi i / (n-1) (symmetric form) evaluated in float32, left to right.  One generator, driven by a
// coefficient row per window, reproduces the reference's tables bit for bit: the harmonic's angle is
// ((2h * pi) * i) / (n-1) with the same three roundings, each term is  acc = acc (-/+) (a_h * cos(angle)).
// (Hann is stored as 0.5 - 0.5 cos: scaling by a power of two commutes with rounding, so it equals 0.5 * (1 - cos).)
struct CosineSum {
    int terms;        // harmonics after a0
    float a[4];       // a0, a1, a2, a3 (magnitudes; signs alternate -, +, -)
};

const CosineSum *cosine_sum_for(int window)
{
    static const CosineSum hann{1, {0.5f, 0.5f, 0.0f, 0.0f}};
    static const CosineSum hamming{1, {0.53836f, 0.46164f, 0.0f, 0.0f}};
    static const CosineSum blackman{2, {0.42f, 0.5f, 0.08f, 0.0f}};
    static const CosineSum blackman_harris{3, {0.35875f, 0.48829f, 0.14128f, 0.01168f}};
    switch(window)
    {
    case WF_WINDOW_HAMMING: return &hamming;
    case WF_WINDOW_BLACKMAN: return &blackman;
    case WF_WINDOW_BLACKMAN_HARRIS: return &blackman_harris;
    case WF_WINDOW_POWER_OF_SINE: return nullptr;
    default: return &hann;
    }
}

void build_window(Tables &t)
{
    const size_t n = (size_t)t.N;
    if(t.cfg.window == WF_WINDOW_NONE)
    {
        t.window.clear();
        t.window_sum = (float)n; // a rectangular window sums to n (src/source.cpp:1234)
        return;
    }
    t.window.resize(n);
    const size_t last = n - 1;
    if(const CosineSum *cs = cosine_sum_for(t.cfg.window))
    {
        const float turn[3] = {2 * kPi, 4 * kPi, 6 * kPi}; // 2 pi h, h = 1..3
        for(size_t i = 0; i < n; ++i)
        {
            float acc = cs->a[0];
            for(int h = 0; h < cs->terms; ++h)
            {
                const float term = cs->a[h + 1] * std::cos((turn[h] * i) / last);
                acc = (h & 1) ? acc + term : acc - term;
            }
            t.window[i] = acc;
        }
    }
    else
    {
        const float exponent = (float)t.cfg.sine_exponent;
        for(size_t i = 0; i < n; ++i)
            t.window[i] = std::pow(std::sin((kPi * i) / last), exponent);
    }
    // m_window_sum: one float accumulator, index order (src/source.cpp:1228-1231) — the magnitude normalisation 2/sum
    // must see exactly the reference's rounding
    float total = 0.0f;
    for(float w : t.window)
        total += w;
    t.window_sum = total;
}

// ---- slope: +3 dB-ish per decade tilt, m[i] = log10(10 * 1000^(i*slope/(B-1))) (src/source.cpp:1282-1290) ----------
void build_slope(Tables &t)
{
    t.slope.clear();
    if(!(t.cfg.slope > 0.0f))
        return;
    const size_t bins = (size_t)t.B;
    const float top = (float)(bins - 1);
    t.slope.resize(bins);
    for(size_t k = 0; k < bins; ++k)
        t.slope[k] = std::log10(geo_lerp(10.0f, 10000.0f, ((float)k * t.cfg.slope) / top));
}

// ---- roll-off: rate dB per octave outside [cutoff_low * 2^q, cutoff_high / 2^q] (init_rolloff, src/source.cpp:898-918) ---
void build_rolloff(Tables &t)
{
    t.rolloff.clear();
    const auto &c = t.cfg;
    if(!((c.rolloff_q > 0.0f) && (c.rolloff_rate > 0.0f)))
        return;
    const float hz_per_bin = (float)c.sample_rate / (float)(size_t)t.N;
    const float shrink = std::exp2(c.rolloff_q);
    const float knee_lo = (float)c.cutoff_low * shrink;
    const float knee_hi = (float)c.cutoff_high / shrink;
    // attenuation for a frequency that lies `r` times beyond a knee (r <= 1: inside the pass band)
    auto beyond = [&](float r) { return (r > 1.0f) ? (c.rolloff_rate * std::log2(r)) : 0.0f; };
    t.rolloff.assign((size_t)t.B, 0.0f); // bin 0 is never attenuated
    for(size_t k = 1; k < (size_t)t.B; ++k)
    {
        const float hz = k * hz_per_bin;
        t.rolloff[k] = beyond(knee_lo / hz) + beyond(hz / knee_hi);
    }
}

// ---- interpolation kernels: per display point, the taps' weights for the bins around floor(x) ---------------------
// Catmull-Rom with tension tau (make_catrom_kernel, src/filter.hpp:67-103): tap j's weight is a cubic in the
// fractional position u; basis[j] holds its coefficients for u^0..u^3, evaluated as a plain ascending dot product
// starting from 0 (the rounding sequence the reference's matrix product has).
void build_catrom(Tables &t, float tau)
{
    const float basis[4][4] = {{0, -tau, 2 * tau, -tau}, {1, 0, tau - 3, 2 - tau}, {0, tau, 3 - (2 * tau), tau - 2}, {0, 0, -tau, tau}};
    const size_t points = t.interp_indices.size();
    t.interp_radius = 2;
    t.interp_taps = 4;
    t.interp_weights.assign(points * 4, 0.0f);
    for(size_t pt = 0; pt < points; ++pt)
    {
        const float u = t.interp_indices[pt] - std::floor(t.interp_indices[pt]);
        const float powers[4] = {1, u, u * u, u * u * u};
        for(int tap = 0; tap < 4; ++tap)
        {
            float w = 0;
            for(int e = 0; e < 4; ++e)
                w += powers[e] * basis[tap][e];
            t.interp_weights[pt * 4 + tap] = w;
        }
    }
}

// Lanczos window of half-width a (make_lanczos_kernel, src/filter.hpp:106-131; sinc / lanczos src/math_funcs.hpp:37-52):
// L(d) = sinc(d) sinc(d/a) for |d| < a, taps at the 2a integer bins (int)x - a + 1 ... (int)x + a.
void build_lanczos(Tables &t, int a)
{
    auto sinc = [](float v) {
        if(v == 0.0)
            return 1.0f;
        const auto pv = kPi * v;
        return std::sin(pv) / pv;
    };
    const size_t points = t.interp_indices.size();
    const int taps = 2 * a;
    const float width = (float)a;
    t.interp_radius = a;
    t.interp_taps = taps;
    t.interp_weights.assign(points * (size_t)taps, 0.0f);
    for(size_t pt = 0; pt < points; ++pt)
    {
        const float x = t.interp_indices[pt];
        const intmax_t first = (intmax_t)x - a + 1;
        for(int tap = 0; tap < taps; ++tap)
        {
            const float d = x - (first + tap);
            t.interp_weights[pt * (size_t)taps + tap] = (std::abs(d) < width) ? sinc(d) * sinc(d / width) : 0.0f;
        }
    }
}

// init_interp, src/source.cpp:837-896 (spectrum display modes only)
void build_interp(Tables &t, unsigned sz)
{
    const auto &c = t.cfg;
    const size_t fft_size = (size_t)t.N;
    const auto maxbin = (fft_size / 2) - 1;
    const auto sr = (float)c.sample_rate;
    const float lowbin = std::clamp((float)c.cutoff_low * fft_size / sr, 1.0f, (float)maxbin);
    const float highbin = std::clamp((float)c.cutoff_high * fft_size / sr, 1.0f, (float)maxbin);

    t.interp_indices.resize(sz);
    for(auto i = 0u; i < sz; ++i)
    {
        const float pos = (c.mirror_freq_axis ? i * 2.0f : (float)i) / (float)(sz - 1);
        const float v = c.log_scale ? geo_lerp(lowbin, highbin, pos) : std_lerp(lowbin, highbin, pos);
        t.interp_indices[i] = std::clamp(v, lowbin, highbin);
    }

    const bool bars = (c.display_mode == WF_DISPLAY_BAR);
    t.band_widths.clear();
    t.band_offsets.clear();
    if(bars)
    {
        t.band_widths.resize((size_t)t.num_bars);
        for(auto i = 0; i < t.num_bars; ++i)
            t.band_widths[i] = std::max((int)(t.interp_indices[i + 1] - t.interp_indices[i]), 1);
        t.band_offsets.resize((size_t)t.num_bars + 1);
        int32_t acc = 0;
        for(auto i = 0; i < t.num_bars; ++i)
        {
            t.band_offsets[i] = acc;
            acc += t.band_widths[i];
        }
        t.band_offsets[t.num_bars] = acc;
    }

    t.interp_weights.clear();
    t.interp_radius = 0;
    t.interp_taps = 0;
    if(c.interp_mode != WF_INTERP_POINT)
    {
        if(bars)
        {
            // m_interp_indices so far holds band starts; fill in every sample point of every band (:876-889)
            std::vector<float> samples;
            for(auto i = 0; i < t.num_bars; ++i)
            {
                auto count = t.band_widths[i];
                for(auto j = 0; j < count; ++j)
                    samples.push_back(t.interp_indices[i] + j);
            }
            t.interp_indices = std::move(samples);
        }
        if(c.interp_mode == WF_INTERP_LANCZOS)
            build_lanczos(t, 4);
        else
            build_catrom(t, 0.5f);
    }
}

// make_gauss_kernel, src/filter.hpp:40-65
void build_gauss(Tables &t)
{
    t.gauss.clear();
    t.gauss_radius = 0;
    t.gauss_sum = 0.0f;
    if(t.cfg.filter_mode != WF_FILTER_GAUSS)
        return;
    float sigma = std::max(std::abs(t.cfg.filter_radius), 0.01f);
    auto w = (int)std::ceil(3.0f * sigma);
    auto size = (2 * w) - 1;
    t.gauss.resize((size_t)size);
    t.gauss_radius = w;
    constexpr auto pi2 = kPi * 2.0f;
    const auto sigsqr = sigma * sigma;
    const auto expdenom = 2.0f * sigsqr;
    const auto coeff = (1.0f / (std::sqrt(pi2) * sigma));
    auto j = 0;
    for(auto i = -w + 1; i < w; ++i)
    {
        auto exponent = -((i * i) / expdenom);
        auto weight = coeff * std::exp(exponent);
        t.gauss[j++] = weight;
        t.gauss_sum += weight;
    }
}

void build_twiddles(Tables &t)
{
    const int M = t.N / 2;
    t.tw.resize((size_t)M * 2);
    t.tw_post.resize((size_t)M * 2);
    for(int k = 0; k < M; ++k)
    {
        const double a = -2.0 * std::numbers::pi * (double)k / (double)M;
        t.tw[2 * k] = (float)std::cos(a);
        t.tw[2 * k + 1] = (float)std::sin(a);
        const double b = -2.0 * std::numbers::pi * (double)k / (double)t.N;
        t.tw_post[2 * k] = (float)std::cos(b);
        t.tw_post[2 * k + 1] = (float)std::sin(b);
    }
}

} // namespace

// std::lerp(float, float, float) as evaluated by libstdc++ (P0811R3 algorithm); the reference's lerp()
// (src/math_funcs.hpp:31-35) forwards to it.
float std_lerp(float a, float b, float t)
{
    if((a <= 0 && b >= 0) || (a >= 0 && b <= 0))
        return t * b + (1 - t) * a;
    if(t == 1)
        return b;
    const float x = a + t * (b - a);
    return ((t > 1) == (b > a)) ? (b < x ? x : b) : (b > x ? x : b);
}

// WAVSource::get_gravity, src/source.hpp:301-312
float gravity_for(const wf_config &c, float seconds)
{
    constexpr float denom = 0.03868924705242879469662125316986f;
    constexpr float hi = denom * 5.0f;
    constexpr float lo = 0.0f;
    if((c.tsmoothing == WF_TSMOOTH_NONE) || (c.gravity <= 0.0f))
        return 0.0f;
    return (c.tsmoothing == WF_TSMOOTH_TVEXPONENTIAL) ? std::exp(-seconds / std_lerp(lo, hi, c.gravity)) : c.gravity;
}

int build_tables(const wf_config &cfg_in, Tables &t, const char **why)
{
    t = Tables{};
    t.cfg = cfg_in;
    auto &c = t.cfg;
    auto fail = [&](const char *msg) {
        if(why)
            *why = msg;
        return (int)WF_ERR_INVALID_ARG;
    };

    // get_settings clamps, src/source.cpp:562-577
    if(c.fft_size < 128)
        c.fft_size = 128;
    else if(c.fft_size & 15)
        c.fft_size &= -16;
    if((c.cutoff_high - c.cutoff_low) < 0)
    {
        c.cutoff_high = 17500;
        c.cutoff_low = 120;
    }
    if((c.ceiling_db - c.floor_db) < 1)
    {
        c.ceiling_db = 0;
        c.floor_db = -120;
    }
    if(c.capture_channels < 1 || c.capture_channels > 2)
        return fail("capture_channels must be 1 or 2 (the plugin captures at most 2, src/source.cpp:1089)");
    if(c.sample_rate == 0)
        return fail("sample_rate must be > 0");
    if(c.max_streams < 1)
        return fail("max_streams must be >= 1");
    if(c.window < WF_WINDOW_NONE || c.window > WF_WINDOW_POWER_OF_SINE)
        return fail("unknown window");
    if(c.tsmoothing < WF_TSMOOTH_NONE || c.tsmoothing > WF_TSMOOTH_TVEXPONENTIAL)
        return fail("unknown tsmoothing mode");
    if(c.interp_mode < WF_INTERP_POINT || c.interp_mode > WF_INTERP_CATROM)
        return fail("unknown interp_mode");
    if(c.display_mode < WF_DISPLAY_CURVE || c.display_mode > WF_DISPLAY_BAR)
        return fail("unknown display_mode");
    if(c.width < 2 || c.width > 16384)
        return fail("width out of range");
    if(c.display_mode == WF_DISPLAY_BAR && (c.bar_width < 1 || c.bar_gap < 0))
        return fail("bar_width must be >= 1 and bar_gap >= 0");
    c.stereo = c.stereo ? 1 : 0;

    t.N = c.fft_size;
    t.B = t.N / 2;
    t.output_channels = ((c.capture_channels > 1) || c.stereo) ? 2 : 1; // src/source.cpp:1170
    t.display_channels = c.stereo ? 2 : 1;
    t.db_min = 20.0f * std::log10(std::numeric_limits<float>::min()); // src/source.cpp:43

    build_window(t);

    // display points, src/source.cpp:1250-1276
    if(c.display_mode == WF_DISPLAY_CURVE)
    {
        t.num_bars = 0;
        t.num_points = c.width;
        build_interp(t, (unsigned)c.width);
    }
    else
    {
        const auto bar_stride = c.bar_width + c.bar_gap;
        t.num_bars = (int)((unsigned)c.width / (unsigned)bar_stride);
        if(((int)c.width - (t.num_bars * bar_stride)) >= c.bar_width)
            ++t.num_bars;
        if(t.num_bars < 1)
            return fail("width too small for one bar");
        t.num_points = t.num_bars;
        build_interp(t, (unsigned)(t.num_bars + 1)); // extra band for the last bar
    }

    // display geometry, src/source.cpp:579-580 (spacing), :655-656 (caps), :1365-1373 (curve), :1481-1493 (bars)
    if(c.height < 1)
        c.height = 225;
    if(!c.stereo || (c.height - c.channel_spacing) < 1)
        c.channel_spacing = 0;
    if(c.display_mode != WF_DISPLAY_BAR)
        c.rounded_caps = 0;
    {
        const auto center = (float)c.height / 2;
        const auto bottom = (float)c.height;
        const auto cpos = c.stereo ? center : bottom;
        const auto channel_offset = c.channel_spacing * 0.5f;
        t.px_cpos = cpos;
        if(c.display_mode == WF_DISPLAY_CURVE)
        {
            t.px_lo = 0.0f;
            t.px_hi = cpos - channel_offset;
        }
        else
        {
            const float cap_radius = (float)c.bar_width / 2.0f;
            auto border_top = c.rounded_caps ? cap_radius : 0.0f;
            auto border_bottom = (c.rounded_caps && (!c.stereo || (c.channel_spacing > 0))) ? cpos - cap_radius : cpos;
            if(c.channel_spacing > 0)
                border_bottom -= channel_offset;
            if(c.min_bar_height > 0)
                border_bottom -= c.min_bar_height;
            border_bottom = std::clamp(border_bottom, border_top, cpos);
            t.px_lo = border_top;
            t.px_hi = border_bottom;
        }
    }

    build_gauss(t);
    build_slope(t);
    build_rolloff(t);
    build_twiddles(t);
    return WF_OK;
}

int build_wave_tables(const wf_wave_config &w, Tables &t, const char **why)
{
    t = Tables{};
    auto fail = [&](const char *msg) {
        if(why)
            *why = msg;
        return (int)WF_ERR_INVALID_ARG;
    };
    if(w.width < 2)
        return fail("the waveform display stage needs width >= 2");
    if(w.interp_mode < WF_INTERP_POINT || w.interp_mode > WF_INTERP_CATROM)
        return fail("unknown interp_mode");
    auto &c = t.cfg;
    c.display_mode = WF_DISPLAY_CURVE;
    c.width = w.width;
    c.stereo = w.stereo ? 1 : 0;
    c.interp_mode = w.interp_mode;
    c.filter_mode = w.filter_mode;
    c.filter_radius = w.filter_radius;
    c.height = w.height;
    c.floor_db = w.floor_db;
    c.ceiling_db = w.ceiling_db;
    c.channel_spacing = w.channel_spacing;
    // get_settings clamps, src/source.cpp:573-580
    if((c.ceiling_db - c.floor_db) < 1)
    {
        c.ceiling_db = 0;
        c.floor_db = -120;
    }
    if(c.height < 1)
        c.height = 225;
    if(!c.stereo || (c.height - c.channel_spacing) < 1)
        c.channel_spacing = 0;

    t.N = c.width; // m_fft_size := m_width, src/source.cpp:1140
    t.num_points = c.width;
    t.display_channels = c.stereo ? 2 : 1;
    t.db_min = 20.0f * std::log10(std::numeric_limits<float>::min());

    // init_interp(m_width), src/source.cpp:842-846 and :859-863 (m_log_scale and m_mirror_freq_axis forced off, :1136-1137)
    const unsigned sz = (unsigned)c.width;
    const float lowbin = 0.0f, highbin = (float)(sz - 1);
    t.interp_indices.resize(sz);
    for(auto i = 0u; i < sz; ++i)
        t.interp_indices[i] = std::clamp(std_lerp(lowbin, highbin, (float)i / (float)(sz - 1)), lowbin, highbin);
    t.interp_weights.clear();
    if(c.interp_mode == WF_INTERP_LANCZOS)
        build_lanczos(t, 4);
    else if(c.interp_mode == WF_INTERP_CATROM)
        build_catrom(t, 0.5f);
    build_gauss(t);

    // render_curve geometry, src/source.cpp:1368-1373, 1410
    const auto cpos = c.stereo ? (float)c.height / 2 : (float)c.height;
    t.px_cpos = cpos;
    t.px_lo = 0.0f;
    t.px_hi = cpos - c.channel_spacing * 0.5f;
    return WF_OK;
}

} // namespace wf
