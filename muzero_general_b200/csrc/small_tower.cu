// Fused CUDA-core residual tower (small_tower.h).
//
// The per-layer conv3x3_kernel (resnet.cu) is latency-bound on small boards: a TicTacToe / Breakout-hidden conv is
// 20-340 MFLOP per launch, far too little to amortise a launch, the weight staging and the input staging, and a
// simulation needs 5-9 of them.  Here ONE persistent launch runs the whole tower: every CTA stages the weights of all
// layers once, then takes tiles of `boards_per_cta` boards through all layers with the activations ping-ponging
// between two zero-padded shared-memory buffers; only the tower input is read from and the tower output written to
// global memory.  A residual block (models.py:213-231) is conv1: X -> T, conv2: T -> X with the residual X added in
// place by the thread that owns the output.  The arithmetic (fp32 FMA chain over cin, dy, dx; + bias, + residual,
// ReLU) is in exactly the order of conv3x3_kernel, so both paths give bit-identical results.
//
// Thread mapping: one item = (board, row y, row segment, group of CO output channels) computes P consecutive pixels of
// that row for CO channels (P x CO accumulators; P = W, or W/2 for small latency-bound batches); CO = 4 when the batch is large enough to fill the GPU that way (float4
// weight loads, 4.5+ FMAs per shared-memory load), CO = 1 for small batches (4x the threads, lower latency).
#include "small_tower.h"
#include "small_tower.cuh"
#include "launch.h"

#include <algorithm>

namespace mz {

namespace {
constexpr int kMaxThreads = 704;      // 22 warps: one CTA can hold a whole SM's share of a large batch (weights staged once per SM)

template <int P, int CO>
__global__ void __launch_bounds__(kMaxThreads) small_tower_kernel(const __grid_constant__ SmallTowerArgs a) {
    extern __shared__ __align__(16) float smem[];
    float* s_w = smem;
    float* s_act = smem + a.w_floats;
    // ---- once per CTA: weights + biases of every layer, zeroed activation buffers (padding stays zero)
    pdl_launch_dependents();
    small_tower_stage(a, s_w, s_act, threadIdx.x, blockDim.x);
    pdl_wait();                                            // weights are constants; the input comes from the previous kernel
    const int nb = a.boards_per_cta;
    for (int tile = blockIdx.x; tile * nb < a.n; tile += gridDim.x)
        small_tower_tile<P, CO, false>(a, s_w, s_act, tile * nb, min(nb, a.n - tile * nb), threadIdx.x, blockDim.x);
}

}  // namespace

// Shared-memory layout of the tower's weights (w_smem_off / b_smem_off / w_floats) and the channel capacity of its
// activation buffers; false (with the reason in *why) when the shape is outside what the kernels handle.
bool small_tower_layout(SmallTowerArgs& a, const char** why) {
    const char* dummy;
    if (!why) why = &dummy;
    if (a.n_layers < 1 || a.n_layers > kSmallTowerMaxLayers) { *why = "1 to 10 layers"; return false; }
    if (a.W < 2 || a.W > 8 || a.H < 1 || a.H > 16) { *why = "boards of 1..16 rows x 2..8 columns"; return false; }
    if (a.C % 4 != 0 || a.C < 4) { *why = "channels must be a positive multiple of 4"; return false; }
    int cap = a.C, w_floats = 0;
    for (int l = 0; l < a.n_layers; ++l) {
        cap = std::max(cap, a.layer[l].cin);
        a.w_smem_off[l] = w_floats; w_floats += a.layer[l].cin * 9 * a.C;
        a.b_smem_off[l] = w_floats; w_floats += a.C;
    }
    if (a.layer[0].cin != a.in_channels + (a.action ? 1 : 0)) { *why = "the first layer does not read the tower input"; return false; }
    a.cap_channels = cap; a.w_floats = w_floats;
    a.row_stride = a.W + 2; a.board_stride = cap * (a.H + 2) * (a.W + 2);
    return true;
}

namespace {

// false (with the reason in *why) when the fused tower cannot take the shape
bool make_plan(SmallTowerArgs& a, int sm_count, SmallTowerPlan& pl, const char** why) {
    pl = SmallTowerPlan{};
    if (a.n < 1) { *why = "empty batch"; return false; }
    if (!small_tower_layout(a, why)) return false;
    const int cap = a.cap_channels, w_floats = a.w_floats;
    const int plane = (a.H + 2) * (a.W + 2);
    // CO = 4 only when that still gives every SM a few hundred threads
    int CO = ((long)a.n * (a.C / 4) * a.H >= (long)sm_count * 384) ? 4 : 1;
    if ((a.C / CO) * a.H > kMaxThreads) CO = 4;
    // small batches (CO = 1) are latency-bound: split the rows in two segments so twice as many threads share a board
    int P = a.W;
    if (CO == 1 && a.W >= 4 && a.W % 2 == 0 && (a.C / CO) * a.H * 2 <= kMaxThreads) P = a.W / 2;
    const int items = (a.C / CO) * a.H * (a.W / P);
    if (items > kMaxThreads) { *why = "one board needs more threads than a CTA holds"; return false; }
    auto bytes = [&](int boards) { return ((size_t)w_floats + 2ull * boards * cap * plane) * 4; };
    // c CTAs per SM, each with as many boards as its threads and its share of shared memory allow: take the split that
    // keeps most of an SM's share of the batch in flight at once (ties: fewer CTAs, the weights are staged per CTA)
    const size_t smem_cap = 226 * 1024;
    const int want = (a.n + sm_count - 1) / sm_count;
    int best_c = 0, best_nb = 0, best_cover = -1;
    for (int c = 1; c <= 4; ++c) {
        int nb_c = std::min(std::min(kMaxThreads / items, a.n), 2048 / c / items);
        while (nb_c >= 1 && (bytes(nb_c) + 1024) * c > smem_cap) --nb_c;
        if (nb_c < 1) break;
        const int cover = std::min(c * nb_c, want);
        if (cover > best_cover) { best_cover = cover; best_c = c; best_nb = nb_c; }
    }
    if (best_c == 0) { *why = "the weights and one board exceed shared memory"; return false; }
    // persistent grid; spread the boards evenly over the resident CTAs
    int nb = best_nb;
    int grid = sm_count * best_c;
    const int rounds = (a.n + grid * nb - 1) / (grid * nb);
    nb = std::min(nb, (a.n + grid * rounds - 1) / (grid * rounds));
    grid = std::min((a.n + nb - 1) / nb, grid);
    a.boards_per_cta = nb; a.cap_channels = cap; a.w_floats = w_floats;
    pl.P = P; pl.CO = CO; pl.boards_per_cta = nb; pl.threads = ((nb * items + 31) / 32) * 32; pl.grid = grid; pl.smem = bytes(nb);
    return true;
}

template <int P, int CO>
cudaError_t launch(const SmallTowerArgs& a, const SmallTowerPlan& pl, cudaStream_t stream) {
    static size_t attr = 0;
    if (attr < pl.smem) {
        cudaError_t e = cudaFuncSetAttribute(small_tower_kernel<P, CO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
        if (e != cudaSuccess) return e;
        attr = pl.smem;
    }
    cudaError_t e = launch_chained(small_tower_kernel<P, CO>, dim3(pl.grid), dim3(pl.threads), pl.smem, stream, a);
    return e != cudaSuccess ? e : cudaGetLastError();
}
}  // namespace

bool small_tower_supported(const SmallTowerArgs& a) {
    SmallTowerPlan pl;
    return small_tower_plan(a, 132, &pl, nullptr);      // (whether a plan exists does not depend on the SM count)
}

bool small_tower_plan(SmallTowerArgs a, int sm_count, SmallTowerPlan* plan, const char** why) {
    const char* dummy;
    return make_plan(a, sm_count, *plan, why ? why : &dummy);
}

cudaError_t launch_small_tower(SmallTowerArgs a, int sm_count, cudaStream_t stream, SmallTowerPlan* used) {
    SmallTowerPlan pl;
    const char* why;
    if (!make_plan(a, sm_count, pl, &why)) return cudaErrorInvalidValue;
    if (used) *used = pl;
#define MZ_ST(PP)                                                                             \
    if (pl.P == PP) return pl.CO == 4 ? launch<PP, 4>(a, pl, stream) : launch<PP, 1>(a, pl, stream);
    MZ_ST(2) MZ_ST(3) MZ_ST(4) MZ_ST(5) MZ_ST(6) MZ_ST(7) MZ_ST(8)
#undef MZ_ST
    return cudaErrorInvalidValue;
}

}  // namespace mz
