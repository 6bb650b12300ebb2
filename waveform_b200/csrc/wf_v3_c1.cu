// wf_v3_c1.cu — stft_v3_kernel instantiations for one capture channel + the host-side helpers of wf_v3.hpp
#include <cmath>
#include <numbers>

#include "wf_v3_impl.cuh"

namespace wf {

cudaError_t v3_launch_c2(int N, int R, int extra, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display,
                         int device);
cudaError_t v3_launch_s16(int N, int cc, int R, int extra, const KParams &kp, const v3::Tw3 &tw, cudaStream_t st, bool display,
                          int device);

bool v3_supported(int N) { return N == 1024 || N == 2048 || N == 4096 || N == 8192 || N == 16384; }
int v3_min_cluster(int N) { return (N <= 8192) ? 1 : 2; }

size_t v3_smem_bytes(int N, int dch, int n_points, bool display, int cc, int R)
{
    switch(N)
    {
    case 1024: return v3::smem_bytes<1024>(dch, n_points, display, cc, R);
    case 2048: return v3::smem_bytes<2048>(dch, n_points, display, cc, R);
    case 4096: return v3::smem_bytes<4096>(dch, n_points, display, cc, R);
    case 8192: return v3::smem_bytes<8192>(dch, n_points, display, cc, R);
    case 16384: return v3::smem_bytes<16384>(dch, n_points, display, cc, R);
    default: return 0;
    }
}

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

cudaError_t v3_launch(int N, int cc, int R, int extra, bool s16, const KParams &kp, const float *d_tw1, const float *d_tw2,
                      const float *d_tw0, cudaStream_t st, bool display, int device)
{
    v3::Tw3 tw{reinterpret_cast<const float2 *>(d_tw1), reinterpret_cast<const float2 *>(d_tw2),
               reinterpret_cast<const float2 *>(d_tw0)};
    if(s16)
        return v3_launch_s16(N, cc, R, extra, kp, tw, st, display, device);
    if(cc == 2)
        return v3_launch_c2(N, R, extra, kp, tw, st, display, device);
    return v3impl::launch_cc<1, float>(N, R, extra, kp, tw, st, display, device);
}

} // namespace wf
