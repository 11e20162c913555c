// 128-channel residual towers on the tensor cores at fp32-grade accuracy, dense NCHW fp32 in and out (conv_wide.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mz {

constexpr int kWideC = 128;
constexpr int kWideMaxLayers = 21;          // a stem + 10 residual blocks (Gomoku's dynamics tower is 13 layers)

struct WideLayer {
    const float* w;               // x3 image [9 taps][2 K-halves][256 rows: w_h cout 0..127 | w_l cout 0..127][64 cin] fp16,
                                  // 128B-swizzled (typed float*): w = (w_h + w_l) / s, s a power of two per output channel
    const float* scale;           // [128] 1 / s
    const float* bias;            // [128] folded BN shift, or nullptr
    const float* action_table;    // dynamics stem: add (action/A) * table[y * W + x][cout]; nullptr otherwise
};

// [stem conv +] residual blocks of 128 channels, every conv followed by bias (+ residual) (+ action term) + ReLU
struct WideTowerArgs {
    const float* in;              // [n][128][H][W] dense fp32, or the hidden-state pool when gather_parent is set
    float* out;                   // [n][128][H][W]
    const int32_t* gather_parent; // board g reads in + (g * pool_stride + gather_parent[g]) * 128 * H * W
    int pool_stride;
    const int32_t* action;        // [n] for a stem with an action table
    int n, H, W, A;
    int g0;                       // boards [g0, g0 + n): every array is addressed by the global index
    int stem;                     // layer 0 is a stem; the layers after it are blocks of two convs
    int n_layers;
    WideLayer layer[kWideMaxLayers];
    int* sat_count;               // bumped when an activation read or stored exceeds the fp16 range
    // filled by the launcher from the plan
    int S, plane_bytes, res_off, bar_off;
};

// Launch plan of one wide tower (host only; the launchers, mz_debug_wide_tower_plan and mz_debug_wide_pair_tower_plan take it
// from here).  On CTA pairs every per-CTA field describes one CTA holding pair_rows0 = ceil(H / 2) board rows.
struct WideTowerPlan {
    int m_tiles, threads;         // 64-row M-tiles of the (per-CTA) board rows x (W + 1), one warpgroup each
    int rows;                     // shared-memory rows of one activation plane (guard + zero rows + board, multiple of 8)
    int stages;                   // weight ring stages (one tap x one 64-channel K-half each)
    size_t smem;                  // dynamic shared-memory bytes
    int layers;
    int ctas_per_sm, wave;        // resident CTAs per SM; boards per wave on the device (CTA pairs: ctas_per_sm x SMs / 2)
    int launches;                 // kernel launches per tower call
    int reg_cap;                  // registers per thread the plan assumes (__launch_bounds__ of the kernel)
    int pair_rows0;               // CTA pairs: board rows of CTA 0 (CTA 1 takes the rest); 0 on the one-CTA route
};

// false with the reason in *why when the wide tower refuses the shape (the network then keeps the CUDA-core towers)
bool wide_tower_plan(int n, int C, int H, int W, int layers, int sm_count, WideTowerPlan* p, const char** why);
cudaError_t launch_wide_tower(WideTowerArgs a, const WideTowerPlan& p, cudaStream_t stream);
// The same tower with each board split across a cluster of two CTAs (rows [0, pair_rows0) and the rest), for boards one CTA
// cannot hold (15 x 15, 16 x 16); it accepts every board with H >= 2 whose half fits the one-CTA budget.
bool wide_pair_plan(int n, int C, int H, int W, int layers, int sm_count, WideTowerPlan* p, const char** why);
cudaError_t launch_wide_pair_tower(WideTowerArgs a, const WideTowerPlan& p, cudaStream_t stream);

// 256-channel towers (conv_wide256.cu, MZ_TC_WIDE=3): the output channels split across a CTA pair, several boards stacked
// in the M rows of each CTA.  The layers are WideLayers of a 256-channel x3 image: two 128-output-channel halves, each
// [9 taps][4 K-quarters][256 rows: w_h cout | w_l cout][64 cin] fp16, 128B-swizzled; scale / bias [256]; the dynamics
// stem's table [H * W][256].
constexpr int kWide256C = 256;
constexpr int kWide256MaxLayers = 33;       // a stem + 16 residual blocks (games/atari.py's dynamics tower)

struct Wide256Args {
    const float* in;              // [n][256][H][W] dense fp32, or the hidden-state pool when gather_parent is set
    float* out;                   // [n][256][H][W]
    const int32_t* gather_parent; // board g reads in + (g * pool_stride + gather_parent[g]) * 256 * H * W
    int pool_stride;
    const int32_t* action;        // [n] for a stem with an action table
    int n, H, W, A;
    int g0;                       // boards [g0, g0 + n): every array is addressed by the global index
    int stem;                     // layer 0 is a stem; the layers after it are blocks of two convs
    int n_layers;
    WideLayer layer[kWide256MaxLayers];
    int* sat_count;               // bumped when an activation read or stored exceeds the fp16 range
    // filled by the launcher from the plan
    int S, boards, interior, plane_bytes, res_off, bar_off;
};

// Launch plan of one 256-channel tower (host only).  Every per-CTA field describes one CTA of a pair holding `boards`
// stacked boards and 128 of the output channels.
struct Wide256Plan {
    int boards;                   // boards stacked in the M rows of each CTA pair
    int m_tiles, threads;         // 64-row M-tiles of the (boards (H + 1) - 1) (W + 1) interior rows, one warpgroup each
    int rows, interior;           // shared-memory rows of one activation plane (multiple of 8); interior rows computed
    int stages;                   // weight ring stages (one tap x one 64-channel K-quarter x 128 output channels each)
    size_t smem;                  // dynamic shared-memory bytes per CTA
    int layers;
    int ctas_per_sm, wave;        // resident CTAs per SM; boards per wave (ctas_per_sm x SMs / 2 pairs x boards)
    int launches;                 // kernel launches per tower call
    int reg_cap;                  // registers per thread the plan assumes (__launch_bounds__ of the kernel)
};

// false with the reason in *why when the 256-channel tower refuses the shape; force_boards > 0 plans that many boards per
// CTA pair instead of the largest number that fits
bool wide256_plan(int n, int C, int H, int W, int layers, int sm_count, int force_boards, Wide256Plan* p, const char** why);
cudaError_t launch_wide256_tower(Wide256Args a, const Wide256Plan& p, cudaStream_t stream);

}  // namespace mz
