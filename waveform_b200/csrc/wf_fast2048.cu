// wf_fast2048.cu — instantiations of stft2048_fast_kernel (its own translation unit)
#include <array>
#include <utility>

#include "wf_host.hpp"
#include "wf_fast2048.cuh"
#include "wf_fast2048.hpp"

namespace wf {

// indexed by TSM * 4 + GATE * 2 + EXTRA
template<typename TS, int... I>
static std::array<const void *, sizeof...(I)> kernels(std::integer_sequence<int, I...>)
{
    return {(const void *)stft2048_fast_kernel<fast::kMaxWarpsPerCta, (I & 4) != 0, (I & 2) != 0, (I & 1) != 0, TS>...};
}

KernelRef fast2048_kernel(bool tsm, bool gate, bool extra, bool s16)
{
    static const std::array table = {kernels<float>(std::make_integer_sequence<int, 8>{}),
                                     kernels<int16_t>(std::make_integer_sequence<int, 8>{})};
    return {table[s16][tsm * 4 + gate * 2 + extra], fast::kMaxWarpsPerCta * 32, (size_t)fast::smem_bytes(fast::kMaxWarpsPerCta)};
}

} // namespace wf
