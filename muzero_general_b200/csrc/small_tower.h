// Fused CUDA-core residual tower for small boards / few channels (TicTacToe 3x3x16, Breakout's 6x6x16 hidden
// board ...): [optional stem conv] + residual blocks (models.py:206-231) in ONE launch, fp32, a board's
// activations stay in shared memory through all the layers (small_tower.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mz {

constexpr int kSmallTowerMaxLayers = 10;

struct SmallTowerLayer {
    int w_off, b_off;        // into the conv blob: weights [cin][9][C], folded BN bias [C] (b_off < 0: none)
    int cin;                 // input channels (C, or C+1 with the action plane, or the observation channels)
    int residual;            // 1: add the previous content of the output buffer (the block input) before the ReLU
    int relu;
};

struct SmallTowerArgs {
    const float* in;         // [n][in_channels][H][W] dense fp32, or the hidden pool when gather_parent is set
    float* out;              // [n][C][H][W]
    const float* blob;       // conv blob (weights + biases)
    const int32_t* gather_parent;   // sample g reads in + (g*pool_stride + gather_parent[g]) * in_channels*H*W
    const int32_t* action;   // [n]: constant plane action/A appended as channel in_channels (dynamics stem), or nullptr
    int pool_stride;
    int n, C, H, W, A;
    int g0;                  // boards [g0, g0 + n): in / out / action / gather_parent are addressed by the global index
    int in_channels;         // channels of `in` as stored (without the action plane)
    int n_layers;
    SmallTowerLayer layer[kSmallTowerMaxLayers];
    // filled by the launcher
    int boards_per_cta, cap_channels, w_floats;
    int row_stride;          // floats between the rows of a padded plane (W + 2, or W + 3 to make it odd: see small_tower.cuh)
    int board_stride;        // floats between the boards of an activation buffer (>= cap_channels * (H + 2) * row_stride)
    int w_smem_off[kSmallTowerMaxLayers], b_smem_off[kSmallTowerMaxLayers];
};

// Launch of small_tower_kernel<P, CO>: P pixels and CO output channels per thread, boards per CTA, threads per CTA,
// persistent grid (a CTA takes tiles grid apart) and dynamic shared memory
struct SmallTowerPlan { int P, CO, boards_per_cta, threads, grid; size_t smem; };

// fills cap_channels, w_floats, w_smem_off, b_smem_off and the plain strides (row W + 2, board cap * plane); false (with
// the reason in *why, when given) when the shape is outside what the kernels handle
bool small_tower_layout(SmallTowerArgs& a, const char** why = nullptr);
// true when the whole tower (all weights + two activation buffers of a board tile) fits on chip
bool small_tower_supported(const SmallTowerArgs& a);
// the plan launch_small_tower takes for `a` on sm_count SMs (host only); false with the reason in *why when the fused
// tower refuses the shape
bool small_tower_plan(SmallTowerArgs a, int sm_count, SmallTowerPlan* plan, const char** why);
// `used`, when given, receives the plan of the launch
cudaError_t launch_small_tower(SmallTowerArgs a, int sm_count, cudaStream_t stream, SmallTowerPlan* used = nullptr);

}  // namespace mz
