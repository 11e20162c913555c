// wgmma implicit-GEMM conv3x3 on the P64C8 fp16 board layout (conv_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mz {

constexpr int kTowerMaxLayers = 8;
constexpr int kTowerMaxTiles = 8;          // tiles (pairs of boards) one CTA may own in the fused-tower mode
constexpr int kTowerBuffers = 5;

// One conv3x3 (+bias, +residual, +action term, +ReLU) of a tower; buffers are indices into TowerArgs::buf.
struct TowerLayer {
    const float* w;               // fp16 image [9][cout 64][cin 64], 128B-swizzled (typed float*), BN scale folded;
                                  // x3 mode: [9][w_h couts | w_l couts = 128 rows][cin 64] (conv_x3.cu)
    const float* bias;            // [64] folded BN shift, or nullptr
    const float* scale;           // x3 mode: [64] power of two that undoes the per-output-channel weight prescale
    const float* action_table;    // dynamics stem: add (action/A) * table[p][cout]; nullptr otherwise
    int in_buf, out_buf, res_buf; // res_buf = -1: no residual
    int relu;
};

// A whole residual tower executed by ONE persistent launch: every CTA keeps its own tiles through all the
// layers (a conv only needs the board itself: padding is zero), the 9 weight-tap slots in shared memory are
// refilled for layer l+1 while the last tile of layer l is still multiplying, and activations round-trip
// through L2 between layers.  n_layers = 1 is the plain single convolution.
struct TowerArgs {
    int n_layers;
    TowerLayer layer[kTowerMaxLayers];
    float* buf[kTowerBuffers];    // activation buffers, fp16 P64S [n][64 pos][64 ch swizzled] (typed float*); buf[0] may be a gathered pool
    const int32_t* gather_parent; // buf[0] of game g = buf[0] + (g*pool_stride + gather_parent[g]) boards
    int pool_stride;
    const int32_t* action;        // [n] for layers with an action_table
    int n, H, W, A;
    int debug_skip;               // profiling only: 1 = no MMA, 2 = no A-tile loads, 4 = no global stores, 8 = no residual loads
    int g0;                       // x3 mode: first board of this launch (a batch is split into launches of <= 4 boards per SM)
    int* sat_count;               // x3 mode: bumped when a stored activation exceeds the fp16 range (accuracy contract left)
    long long* timeline;          // x3 mode, profiling only (MZ_X3_TIMELINE): CTA 0 records clock64 per (layer, tile):
                                  // [0] MMA issue starts, [1] issued, [2] epilogue sees the accumulator, [3] tile rewritten
};

cudaError_t launch_conv_tower_tc(const TowerArgs& a, int sm_count, cudaStream_t stream);
// the same towers at fp32-grade accuracy: split operands, three partial products (conv_x3.cu); any batch size
cudaError_t launch_conv_tower_x3(const TowerArgs& a, int sm_count, cudaStream_t stream);
int conv_x3_launches(int n, int sm_count);
bool conv_tc_supported(int C, int H, int W);
int conv_tc_board_elems(bool split = false);   // float slots per stored board: 2048 (fp16 plane) or 4096 (x_h | x_l planes)
int conv_tc_max_boards_fused(int sm_count);   // largest batch the fused-tower mode handles in one launch

}  // namespace mz
