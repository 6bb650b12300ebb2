// wf_render.hpp — host interface of the render kernel (wf_render.cu): the display stage run on dB rows a caller passes in
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace wf {
struct KParams;

// What one render launch works on: rows of [dch][B] floats, row r = (stream r / n_frames, tick r % n_frames).
struct RenderArgs {
    float *db;          // [rows][dch][B] (device)
    const float *peak;  // [n_frames] or null: gain[t] = min(target_db - peak[t], max_gain) added to bins k >= 1
    float target_db, max_gain;
    int write_db;       // store the normalised rows back into db
    int display;        // points, pixels or minimum requested (else the call only normalises the rows)
    long long rows;
    int n_frames, B, len; // len = dch * B
    int vec4;           // db is 16-byte aligned: 128-bit loads and stores
    int tab_smem;       // the setup tables are copied into shared memory once per CTA
    int row_smem;       // each group's dB row lives in shared memory (else in `scratch`)
    int tab_floats, group_floats; // shared memory: tables, then one area per group
    float *scratch;     // !row_smem: [grid * groups][len] floats
};

// Launch shape of a render call: a warp per row (tn 32) or the whole CTA per row (tn kRenderThreads).
struct RenderPlan {
    int tn = 0, groups = 0, grid = 0;
    size_t smem = 0;
    bool tab_smem = false, row_smem = false;
    int tab_floats = 0, group_floats = 0;
};
constexpr int kRenderThreads = 256;

// Picks the group size from the row length and the number of display points, places tables and rows, and sizes a persistent
// grid.  `kp` carries the display settings (and which outputs are requested).  plan->grid stays 0 when the display scratch
// alone does not fit in shared memory.
cudaError_t render_plan(const KParams &kp, int B, long long rows, int sm_count, int device, RenderPlan *plan);
cudaError_t render_launch(const RenderPlan &plan, const KParams &kp, const RenderArgs &ra, cudaStream_t st, int device);
} // namespace wf
