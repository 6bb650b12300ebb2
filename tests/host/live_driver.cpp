// live_driver: feeds packets / ticks to wfhost::SpectrumSourceCUDA the way OBS would and dumps m_decibels per tick.
// usage: live_driver <pcm.f32> <channels> <samples_per_channel> <fft_size> <packet> <fps> <ticks> <out.f32> [stereo] [normalize_volume] [sample_rate]
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "spectrum_source.hpp"

int main(int argc, char **argv)
{
    if(argc < 9)
        return 2;
    const char *in = argv[1];
    const int cc = atoi(argv[2]);
    const long ns = atol(argv[3]);
    const int N = atoi(argv[4]), packet = atoi(argv[5]), fps = atoi(argv[6]), ticks = atoi(argv[7]);
    const char *out = argv[8];
    const bool stereo = argc > 9 && atoi(argv[9]) != 0;
    const bool normalize = argc > 10 && atoi(argv[10]) != 0;
    const uint64_t sr = argc > 11 ? strtoull(argv[11], nullptr, 10) : 48000ull;
    std::vector<float> pcm((size_t)cc * ns);
    FILE *f = fopen(in, "rb");
    if(!f || fread(pcm.data(), sizeof(float), pcm.size(), f) != pcm.size())
        return 3;
    fclose(f);

    wf_config cfg;
    wf_config_init(&cfg);
    cfg.sample_rate = (uint32_t)sr;
    cfg.fft_size = N;
    cfg.capture_channels = cc;
    cfg.stereo = stereo;
    cfg.normalize_volume = normalize;
    wfhost::SpectrumSourceCUDA src;
    uint64_t now = 10ull * 1000000000ull;
    int rc = src.update(cfg, 0, now);
    if(rc != WF_OK)
    {
        fprintf(stderr, "update failed: %s\n", wf_strerror(rc));
        return 4;
    }
    FILE *fo = fopen(out, "wb");
    const uint64_t tick_ns = 1000000000ull / (uint64_t)fps;
    const uint64_t pkt_ns = (uint64_t)packet * 1000000000ull / sr;
    uint64_t next_pkt = now, audio_clock = now;
    long pos = 0;
    for(int t = 0; t < ticks; ++t)
    {
        now += tick_ns;
        // deliver all packets due before this tick
        while(next_pkt + pkt_ns <= now && pos + packet <= ns)
        {
            next_pkt += pkt_ns;
            const float *chans[2] = {pcm.data() + pos, cc > 1 ? pcm.data() + ns + pos : nullptr};
            src.capture_audio(chans, (uint32_t)packet, audio_clock, next_pkt, false);
            audio_clock += pkt_ns;
            pos += packet;
        }
        rc = src.tick(1.0f / (float)fps, now);
        if(rc != WF_OK)
        {
            fprintf(stderr, "tick failed: %s (%s)\n", wf_strerror(rc), src.last_error());
            return 5;
        }
        for(int c = 0; c < src.display_channels(); ++c)
            fwrite(src.decibels(c), sizeof(float), (size_t)src.bins(), fo);
        unsigned char s = src.last_silent();
        fwrite(&s, 1, 1, fo);
    }
    fclose(fo);
    printf("ok ticks=%d consumed=%ld bins=%d dch=%d\n", ticks, pos, src.bins(), src.display_channels());
    return 0;
}
