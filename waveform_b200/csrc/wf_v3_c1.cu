// wf_v3_c1.cu — stft_v3_kernel instantiations for one capture channel + the host-side helpers of wf_v3.hpp
#include <cmath>
#include <numbers>

#include "wf_v3_impl.cuh"

namespace wf {

template KernelRef v3_kernel<1, float>(int N, int R, int extra, const KParams &kp, bool display);

KernelRef v3_kernel(int N, int cc, int R, int extra, bool s16, const KParams &kp, bool display)
{
    if(s16)
        return (cc == 2) ? v3_kernel<2, int16_t>(N, R, extra, kp, display) : v3_kernel<1, int16_t>(N, R, extra, kp, display);
    return (cc == 2) ? v3_kernel<2, float>(N, R, extra, kp, display) : v3_kernel<1, float>(N, R, extra, kp, display);
}

int v3_min_cluster(int N) { return (N <= 8192) ? 1 : 2; }

template<int NN>
static void build_tw(std::vector<float> &tw1, std::vector<float> &tw2, std::vector<float> &tw0)
{
    // the split plan (16384) runs its sub-FFTs with the half size's tables and adds the radix-2 stage's W_M^(a*TN + t)
    constexpr int N = v3::Geo3<NN>::SPLIT2 ? NN / 2 : NN;
    using G = v3::Geo3<N>;
    tw0.clear();
    if(v3::Geo3<NN>::SPLIT2)
    {
        using GG = v3::Geo3<NN>;
        tw0.resize((size_t)(GG::P / 2) * GG::TN * 2);
        for(int a = 0; a < GG::P / 2; ++a)
            for(int t = 0; t < GG::TN; ++t)
            {
                const double ang = -2.0 * std::numbers::pi * (double)(a * GG::TN + t) / (double)GG::M;
                tw0[2 * ((size_t)a * GG::TN + t)] = (float)std::cos(ang);
                tw0[2 * ((size_t)a * GG::TN + t) + 1] = (float)std::sin(ang);
            }
    }
    tw1.resize((size_t)G::A * G::TN * 2);
    tw2.resize((size_t)G::B * G::C * 2);
    for(int ka = 0; ka < G::A; ++ka)
        for(int t = 0; t < G::TN; ++t)
        {
            const double a = -2.0 * std::numbers::pi * (double)((long long)t * ka) / (double)G::M;
            tw1[2 * ((size_t)ka * G::TN + t)] = (float)std::cos(a);
            tw1[2 * ((size_t)ka * G::TN + t) + 1] = (float)std::sin(a);
        }
    for(int kb = 0; kb < G::B; ++kb)
        for(int c = 0; c < G::C; ++c)
        {
            const double a = -2.0 * std::numbers::pi * (double)(c * kb) / (double)(G::B * G::C);
            tw2[2 * ((size_t)kb * G::C + c)] = (float)std::cos(a);
            tw2[2 * ((size_t)kb * G::C + c) + 1] = (float)std::sin(a);
        }
}

void v3_build_twiddles(int N, std::vector<float> &tw1, std::vector<float> &tw2, std::vector<float> &tw0)
{
    switch(N)
    {
    case 1024: build_tw<1024>(tw1, tw2, tw0); break;
    case 2048: build_tw<2048>(tw1, tw2, tw0); break;
    case 4096: build_tw<4096>(tw1, tw2, tw0); break;
    case 8192: build_tw<8192>(tw1, tw2, tw0); break;
    case 16384: build_tw<16384>(tw1, tw2, tw0); break;
    default: tw1.clear(); tw2.clear(); tw0.clear(); break;
    }
}

} // namespace wf
