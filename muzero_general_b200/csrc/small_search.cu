// Fused search kernel for small residual networks: every simulation of MCTS.run (self_play.py:302-353) in ONE launch.
//
// The step-wise pipeline runs a simulation as five dependent kernels (dynamics tower -> reward head + rescale ->
// prediction tower -> value / policy heads -> tree step).  For a small board each of them is a latency-bound
// launch that re-stages its weights and round-trips its activations through L2, and a search is 5 N of them.  But
// nothing in a simulation couples two games: the tree step of game g needs the network outputs of game g only, the next
// dynamics call the leaf that tree step selected.  So a CTA takes a tile of games through ALL N simulations by itself:
// tower weights, head weights and the activation buffers stay in shared memory for the whole search, the phases of a
// simulation are separated by __syncthreads() instead of kernel boundaries, and nothing is launched or re-staged in
// between; the raw next state goes from the dynamics tower to the reward head, and the rescaled state from there to the
// prediction tower, through the padded shared-memory board buffers (HeadsTile) - global memory only sees the gathered
// parent state, the new pool state, the three network outputs per game and the tree.  The phases ARE the device functions of the stand-alone kernels (small_tower.cuh, heads.cuh,
// tree_step.cuh) applied to the CTA's games, so every value - hidden states, logits, tree statistics, visit counts - is
// bit-identical to the step-wise pipeline (tests/test_resnet_gpu.py::test_fused_small_search_equals_stepwise_pipeline).
#include "small_search.h"

#include <algorithm>

#include "small_tower.cuh"
#include "tree_step.cuh"

namespace mz {

namespace {

constexpr int kSmallSearchThreads = 512;

template <int P, int CO, int G>
__global__ void __launch_bounds__(kSmallSearchThreads) small_search_kernel(const __grid_constant__ SmallSearchArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const int warp = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
    float* s_wd = smem + a.off_wd;
    float* s_wp = smem + a.off_wp;
    float* s_wh = smem + a.off_wh;
    float* s_scratch = smem + a.off_scratch + (size_t)warp * a.scratch_floats;
    float* s_act = smem + a.off_act;

    // ---- once per CTA: everything that is constant during the search
    pdl_launch_dependents();
    small_tower_stage(a.dyn, s_wd, s_act, tid, nthreads);          // (also zeroes both activation buffers: the padding stays zero)
    small_tower_stage(a.pred, s_wp, s_act, tid, nthreads);
    {
        const float4* src = reinterpret_cast<const float4*>(a.heads_dyn.blob + a.heads_lo);
        float4* dst = reinterpret_cast<float4*>(s_wh);
        for (int i = tid; i < a.heads_floats / 4; i += nthreads) dst[i] = src[i];
    }
    // dense element (c, pos) -> offset inside a board's padded tower buffer (map) / inside the heads' [pos][C + 4] tile (xmap)
    int* s_map = reinterpret_cast<int*>(smem + a.off_map);
    int* s_xmap = s_map + a.dyn.C * a.dyn.H * a.dyn.W;
    {
        const int H = a.dyn.H, W = a.dyn.W, C = a.dyn.C, HW = H * W, Wp = a.dyn.row_stride, plane = (H + 2) * Wp;
        for (int i = tid; i < C * HW; i += nthreads) {
            const int c = i / HW, pos = i - c * HW, yy = pos / W, x = pos - yy * W;
            s_map[i] = c * plane + (yy + 1) * Wp + x + 1;
            s_xmap[i] = pos * (C + 4) + c;
        }
    }
    pdl_wait();                                                    // the root step selected the first leaves
    __syncthreads();
    const float* hblob = s_wh - a.heads_lo;                        // hblob[off] addresses the staged head blob

    const int b0 = (int)blockIdx.x * a.tile;                       // my games: [g0 + b0, g0 + b0 + nbt)
    const int nbt = min(a.tile, a.n - b0);
    if (nbt <= 0) return;
    const int N = a.n_sims;
    const int bufsz = a.tile * a.dyn.board_stride, bstride = a.dyn.board_stride;
    for (int sim = 0; sim < N; ++sim) {
        // dynamics (models.py:379-389, 555-599): parent state gathered from the pool + action plane -> raw next state, which
        // stays in its shared-memory buffer
        const int raw = small_tower_tile<P, CO, CO == 4>(a.dyn, s_wd, s_act, b0, nbt, tid, nthreads, s_map, kTileKeepOutput);
        // reward head on the raw state; min-max rescale -> pool slot of this simulation and buffer 0, the prediction tower's input
        for (int s = warp; s < nbt; s += nwarps)
            heads_one_sample<32>(a.heads_dyn, hblob, s_scratch, nullptr, a.g0 + b0 + s, warp, lane, a.first_slot + sim,
                                 HeadsTile{s_act + raw * bufsz + s * bstride, s_act + s * bstride, s_map, s_xmap});
        // prediction (models.py:424-433) on the rescaled state    (the tile call starts with a CTA barrier)
        const int out = small_tower_tile<P, CO, CO == 4>(a.pred, s_wp, s_act, b0, nbt, tid, nthreads, s_map, kTileInputStaged | kTileKeepOutput);
        for (int s = warp; s < nbt; s += nwarps)
            heads_one_sample<32>(a.heads_pred, hblob, s_scratch, nullptr, a.g0 + b0 + s, warp, lane, 0,
                                 HeadsTile{s_act + out * bufsz + s * bstride, nullptr, s_map, s_xmap});
        __syncthreads();
        // expand + backup with these outputs, then select the next leaf (self_play.py:318-353); read-out after the last one.
        // A warp runs while its first group has a game; a group past the tile's last game replays that one (in its warp).
        for (int lg = tid / G; lg - (lane / G) < nbt; lg += nthreads / G)
            tree_step_game<G, true>(a.tree, a.g0 + b0 + min(lg, nbt - 1), lg < nbt, sim + 1, 0, 1, sim + 1 < N ? 1 : 0,
                                    sim + 1 == N ? 1 : 0);
        // (the next dynamics tile starts with a CTA barrier: leaf_parent / leaf_action of every game are visible)
    }
}

template <int P, int CO, int G>
cudaError_t launch_one(const SmallSearchArgs& a, int threads, size_t smem, cudaStream_t stream) {
    static size_t attr = 0;
    if (attr < smem) {
        cudaError_t e = cudaFuncSetAttribute(small_search_kernel<P, CO, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        attr = smem;
    }
    const int grid = (a.n + a.tile - 1) / a.tile;
    cudaError_t e = launch_chained(small_search_kernel<P, CO, G>, dim3(grid), dim3(threads), smem, stream, a);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace

// Thread mapping and tile size.  CO = 4 output channels per thread (uniform-weight mapping, small_tower.cuh) when that still
// gives a CTA >= 128 tower threads, else one channel per thread and half rows (latency-bound small batches); the tile is the
// largest number of games whose activation buffers fit next to the weights, shrunk so that the CTAs of the launch fill whole
// waves of SMs evenly.  Uniform-weight mapping: odd row stride, board stride = H rows (mod 32) - 32 consecutive rows
// (board, y) of a warp then fall into 32 different shared-memory banks.
bool small_search_shape(int H, int W, int C, int A, int n, int sm_count, int tower_floats, int heads_floats, int scratch_floats,
                        int cap_channels, int* P_, int* CO_, int* G_, int* tile_, int* threads_, size_t* smem_, int* row_stride_, int* board_stride_) {
    if (A > 32 || n < 1 || (W != 3 && W != 6) || C % 4 != 0) return false;
    int G = 4;
    while (G < A) G <<= 1;
    if (G != 4 && G != 16) return false;                       // instantiated group widths (Breakout |A| = 4, TicTacToe |A| = 9)
    const size_t cap_bytes = 227 * 1024;
    for (int CO : {4, 1}) {
        const bool uw = CO == 4;
        const int P = (uw || W == 3) ? W : W / 2;
        if (!((P == 3 && (CO == 1 || CO == 4)) || (P == 6 && CO == 4))) continue;
        const int row_stride = uw ? ((W + 2) | 1) : W + 2;
        const int plane = (H + 2) * row_stride;
        int board_stride = cap_channels * plane;
        if (uw) while (board_stride % 32 != (H * row_stride) % 32) ++board_stride;
        const int items = (C / CO) * H * (W / P);
        // threads: what the towers need, and at least one lane group per game so that the tree step is a single pass
        // (and the heads, one warp per sample, get the warps for it)
        auto threads_for = [&](int tile) {
            const int tower = uw ? (C / CO) * ((tile * H + 31) & ~31) : ((tile * items + 31) / 32) * 32;
            return std::max(tower, ((tile * G + 31) / 32) * 32);
        };
        auto bytes = [&](int tile) {
            return ((size_t)tower_floats + heads_floats + (size_t)(threads_for(tile) / 32) * scratch_floats + 2ull * C * H * W + 2ull * tile * board_stride) * 4 + 256;
        };
        int tile = n;
        while (tile >= 1 && (threads_for(tile) > kSmallSearchThreads || bytes(tile) > cap_bytes)) --tile;
        if (tile < 1) continue;
        const long per_round = (long)sm_count * tile;
        const int rounds = (int)((n + per_round - 1) / per_round);
        tile = std::min(tile, (int)((n + (long)sm_count * rounds - 1) / ((long)sm_count * rounds)));
        const int threads = threads_for(tile);
        if (CO == 4 && tile * items < 128) continue;            // too few busy threads per CTA: one channel per thread instead
        *P_ = P; *CO_ = CO; *G_ = G; *tile_ = tile; *threads_ = threads; *smem_ = bytes(tile);
        *row_stride_ = row_stride; *board_stride_ = board_stride;
        return true;
    }
    return false;
}

cudaError_t launch_small_search(SmallSearchArgs a, int P, int CO, int G, int threads, size_t smem, cudaStream_t stream) {
#define MZ_SS(PP, CC, GG) if (P == PP && CO == CC && G == GG) return launch_one<PP, CC, GG>(a, threads, smem, stream);
    MZ_SS(3, 4, 16) MZ_SS(3, 1, 16) MZ_SS(6, 4, 16)
    MZ_SS(3, 4, 4) MZ_SS(3, 1, 4) MZ_SS(6, 4, 4)
#undef MZ_SS
    return cudaErrorInvalidValue;
}

}  // namespace mz
