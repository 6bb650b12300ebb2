// wf_render.cu — the display stage on dB rows a caller passes in (wf_render): curve points / bars, Gaussian, pixel heights,
// mirroring and (miny, minpos) of rows that out_db of earlier calls produced, optionally after the cross-channel peak gain of
// wf_peak_normalize.  The display arithmetic is display_stage_tab (wf_kernels.cuh), the code every spectrum kernel with
// display outputs runs, so a render of a call's own out_db gives that call's display outputs bit for bit.
#include <cuda_runtime.h>

#include <algorithm>

#include "wf_host.hpp"
#include "wf_kernels.cuh"
#include "wf_render.hpp"

namespace wf {

namespace {

// Persistent: group g of CTA b takes rows b*groups + g, then every gridDim.x*groups-th row after it.  A group of TN threads
// (a warp, or the whole CTA) loads its row into its area (shared memory, or its slice of the L2 scratch when a row does not
// fit), adds the peak gain to bins k >= 1 with peak_normalize_kernel's arithmetic, streams the row back when asked, and runs
// the display stage on it.
// Shared memory: [tables (tab_smem)] then per group [dB row (row_smem) | bar samples | points x 2 | arg-min scratch].
template<int TN>
__global__ void __launch_bounds__(kRenderThreads, 4) render_kernel(const __grid_constant__ KParams p,
                                                                const __grid_constant__ RenderArgs ra)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int GROUPS = kRenderThreads / TN;
    const int grp = threadIdx.x / TN, tid = threadIdx.x % TN;
    float *base = reinterpret_cast<float *>(smem_raw);
    DispTab tb{p.interp_idx, p.interp_w, p.band_widths, p.band_offsets, p.gauss_w};
    if(ra.tab_smem)
    {
        tb = stage_display_tables(p, base, threadIdx.x, blockDim.x);
        base += ra.tab_floats;
        __syncthreads();
    }
    const int dch = p.dch, B = ra.B, len = ra.len;
    const bool need_pts = p.filter || (p.out_pixels != nullptr) || (p.out_min != nullptr);
    float *area = base + (size_t)grp * ra.group_floats;
    float *dbs = ra.row_smem ? area : ra.scratch + ((size_t)blockIdx.x * GROUPS + grp) * len;
    float *tmp = area + (ra.row_smem ? len : 0);
    float *pts = tmp + dch * p.n_sample;
    float *red = pts + (need_pts ? 2 * dch * p.n_points : 0);

    for(long long row = (long long)blockIdx.x * GROUPS + grp; row < ra.rows; row += (long long)gridDim.x * GROUPS)
    {
        float *src = ra.db + row * len;
        const bool gain_on = ra.peak != nullptr;
        const float gain = gain_on ? fminf(ra.target_db - ra.peak[row % ra.n_frames], ra.max_gain) : 0.0f;
        if(ra.vec4)
        {
            // B is a multiple of 8, so a float4 never straddles two channels and only its .x can be bin 0
            const float4 *s4 = reinterpret_cast<const float4 *>(src);
            for(int i = tid; i < len / 4; i += TN)
            {
                float4 v = __ldcs(s4 + i);
                if(gain_on)
                {
                    if((4 * i) % B != 0)
                        v.x += gain;
                    v.y += gain;
                    v.z += gain;
                    v.w += gain;
                    if(ra.write_db)
                        __stcs(reinterpret_cast<float4 *>(src) + i, v);
                }
                reinterpret_cast<float4 *>(dbs)[i] = v;
            }
        }
        else
        {
            for(int i = tid; i < len; i += TN)
            {
                float v = __ldcs(src + i);
                if(gain_on)
                {
                    if(i % B != 0)
                        v += gain;
                    if(ra.write_db)
                        __stcs(src + i, v);
                }
                dbs[i] = v;
            }
        }
        if(!ra.display) // write_db alone: the display stage would store points to a null out_points
            continue;
        group_sync<TN>();
        display_stage_tab<TN, false>(p, tb, dbs, pts, tmp, B, dch, (size_t)row, tid, true, red);
        group_sync<TN>(); // the next row may overwrite dbs
    }
}

template<int TN>
size_t render_smem(const RenderPlan &pl)
{
    return ((pl.tab_smem ? (size_t)pl.tab_floats : 0) + (size_t)(kRenderThreads / TN) * pl.group_floats) * sizeof(float);
}

// floats of one group's area, rounded up to 16 bytes
int group_floats(const KParams &kp, int B, int tn, bool row_smem)
{
    const bool need_pts = kp.filter || kp.out_pixels || kp.out_min;
    const size_t f = (row_smem ? (size_t)kp.dch * B : 0) + (size_t)kp.dch * kp.n_sample +
                     (need_pts ? 2 * (size_t)kp.dch * kp.n_points : 0) + 2 * (size_t)tn;
    return (int)((f + 3) & ~(size_t)3);
}

} // namespace

cudaError_t render_plan(const KParams &kp, int B, long long rows, int sm_count, int device, RenderPlan *plan)
{
    *plan = RenderPlan{};
    constexpr size_t kMaxSmem = 227 * 1024; // opt-in shared memory per CTA on sm_90
    RenderPlan pl;
    pl.tab_floats = (int)((display_table_floats(kp) + 3) & ~(size_t)3);
    // A warp per row while a row and its points are a few thousand floats; longer rows would leave the SM with few rows in
    // flight per warp's worth of latency, so the CTA shares each row.
    const bool warp = (size_t)kp.dch * B <= 4096 && (size_t)kp.dch * kp.n_points <= 2048;
    bool found = false;
    for(const int tn : {warp ? 32 : kRenderThreads, kRenderThreads})
    {
        pl.tn = tn;
        pl.groups = kRenderThreads / tn;
        // in order of preference: tables and rows in shared memory, rows only, neither (CTA groups only: the row then
        // goes to the L2 scratch)
        for(const auto &[tab, row] : {std::pair{true, true}, {false, true}, {false, false}})
        {
            if(!row && tn != kRenderThreads)
                break;
            pl.tab_smem = tab;
            pl.row_smem = row;
            pl.group_floats = group_floats(kp, B, tn, row);
            pl.smem = (tn == 32) ? render_smem<32>(pl) : render_smem<kRenderThreads>(pl);
            if(pl.smem <= kMaxSmem)
            {
                found = true;
                break;
            }
        }
        if(found)
            break;
    }
    if(!found)
        return cudaSuccess;
    const void *kernel = (pl.tn == 32) ? (const void *)render_kernel<32> : (const void *)render_kernel<kRenderThreads>;
    if(cudaError_t err = opt_in_smem(kernel, device, pl.smem))
        return err;
    int per_sm = 0;
    if(cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kRenderThreads, pl.smem))
        return err;
    const long long ctas = (rows + pl.groups - 1) / pl.groups;
    pl.grid = (int)std::max<long long>(1, std::min<long long>(ctas, (long long)sm_count * std::max(per_sm, 1)));
    *plan = pl;
    return cudaSuccess;
}

cudaError_t render_launch(const RenderPlan &pl, const KParams &kp, const RenderArgs &ra, cudaStream_t st, int device)
{
    if(pl.tn == 32)
        return launch_kernel(render_kernel<32>, device, pl.grid, kRenderThreads, pl.smem, st, {}, kp, ra);
    return launch_kernel(render_kernel<kRenderThreads>, device, pl.grid, kRenderThreads, pl.smem, st, {}, kp, ra);
}

} // namespace wf
