// conv3x3 (C -> C, stride 1, pad 1) as an implicit GEMM on the Hopper tensor cores (wgmma).
//
// Used for the residual towers of board-sized states (H <= 6, W <= 7, C = 64: Connect4,
// models.py:213-229 inside representation / dynamics / prediction).  Two kernels share the MMA loop:
//
//   conv_tower_resident_kernel   up to 4 tiles per CTA (1056 boards on 132 SMs): the activations of a CTA's tiles stay
//                                in shared memory through all layers of a tower (see the comment above the kernel)
//   conv_tower_tc_kernel         larger batches / single convs: activations stream through L2, per CTA
//
//     weights  [tap 9][cout C][cin C] fp16, BN folded, 128B-swizzled   shared memory (bulk copy)
//     A tile   two boards = 128 rows of the "P64S" layout               one 8 KB cp.async.bulk per board
//     D        64 x 64 fp32 accumulator per board                       registers of the board's warpgroup
//
// Operands are fp16 (10-bit mantissa - the same as tf32 - with fp32 accumulation): one wgmma consumes K = 16
// channels per 32-byte operand row, so a board needs 36 m64n64k16 MMAs per layer, and every activation / weight byte
// moved through L2 and shared memory is half of what a tf32 formulation moves.
//
// P64S activation layout (HBM and shared): a board is 64 positions p = (y+1)*8 + x (row 0, rows H+1.. and columns
// W..7 are zero padding), every position one 128-byte row of 64 fp16 channels whose eight 16-byte chunks are stored
// XOR-ed with p % 8 - i.e. the boards sit in HBM already in the K-major SWIZZLE_128B shared-memory image of a wgmma
// operand, so a plain 1-D bulk copy lands them ready for the tensor core.  Filter tap (dy,dx) is the SAME shared-memory
// tile with its start address moved by (dy*8+dx) rows (the hardware swizzles on absolute address bits): the implicit
// GEMM needs no im2col copy.  The epilogue works on the accumulator registers: folded-BN bias, the optional residual
// and the optional action-plane term (models.py:557-572 folded into a per-position table), ReLU, zero padding
// positions, convert to fp16 (round to nearest, saturating) and store P64S again.
//
// Warp roles: warpgroup b (warps 4b..4b+3) multiplies and finishes board b of every tile (M = 64 = one board), one
// more warp is the bulk-copy producer; the streaming kernel has a further warp for the output bulk stores.
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>

#include "pipeline.h"
#include "conv_tc.h"
#include "launch.h"
#include "tc_common.cuh"

namespace mz {

namespace {

using namespace tc;

constexpr int kC = 64;                 // channels in = out
constexpr int kPos = 64;               // positions per board (8 x 8 padded grid)
constexpr int kBoards = 2;             // boards per tile, one per consumer warpgroup
constexpr int kHalo = 16;              // zero rows above / below the tile (|shift| <= 9; multiple of 8 keeps the swizzle phase)
constexpr int kRows = kBoards * kPos + 2 * kHalo;      // 160 rows
constexpr int kRowBytes = kC * 2;                      // 128 B: one position, 64 fp16 channels = one 128B-swizzle row
constexpr int kStageBytes = kRows * kRowBytes;         // 20480
constexpr int kStages = 2;
constexpr int kTapBytes = kC * kRowBytes;               // 8192: [cout 64][128 B]
constexpr int kWBytes = 9 * kTapBytes;                 // 73728
constexpr int kOutBytes = kBoards * kPos * kRowBytes;  // 16384: one output tile in the global board layout
constexpr int kBoardHalves = kC * kPos;                // 4096 fp16 per board
constexpr int kConsumerWarps = 4 * kBoards;            // two warpgroups
constexpr int kThreads = 32 * kConsumerWarps + 64;     // + producer warp + store warp
constexpr int kThreadsR = 32 * kConsumerWarps + 32;    // resident kernel: + producer warp

struct Smem {
    // offsets
    static constexpr int w = 0;
    static constexpr int a = 2 * kWBytes;                                  // two weight sets: layer l+1 is prefetched while layer l multiplies
    static constexpr int out = a + kStages * kStageBytes;                  // 2 output tiles (2 boards x 8 KB) staged for the bulk store
    static constexpr int bias = out + 2 * kOutBytes;                       // [kTowerMaxLayers][64] floats
    static constexpr int bars = bias + kTowerMaxLayers * kC * 4;           // 8-byte aligned
    static constexpr int total = bars + 64 * 8;
};
static_assert(Smem::total <= 232448, "shared memory budget");

// The 36 MMAs of one board and one layer: D = sum over taps and 16-channel K steps of the shifted board window times
// the tap's weights.  a16 / w16: descriptor low words of the board's row 0 and of tap 0 of the weight set.
MZ_DEVINL void board_conv(float* d, uint32_t a16, uint32_t w16, uint32_t bar_w_full0, int wait_weights, uint32_t w_parity) {
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        if (wait_weights) mbar_wait(bar_w_full0 + 8u * tap, w_parity);
        constexpr int kRow16 = kRowBytes / 16;                       // 8 sixteen-byte units per row
        const int shift = (tap / 3 - 1) * 8 + (tap % 3 - 1);         // compile-time after unrolling
#pragma unroll
        for (int ks = 0; ks < kC / 16; ++ks)                         // K = 16 channels = 32 bytes of the row
            wgmma_m64n64k16(d, a16 + (uint32_t)(shift * kRow16 + ks * 2), w16 + (uint32_t)(tap * (kTapBytes / 16) + ks * 2),
                            (tap | ks) != 0);                        // start addresses < 2^14 units: no carry into the flags
    }
    wgmma_commit();
    wgmma_wait_all();
}

// bias + residual + action term + ReLU of one accumulator pair, packed to fp16x2 (the inputs of a padding position are
// irrelevant: callers store zero there)
MZ_DEVINL uint32_t finish_pair(float d0, float d1, const float* bias, uint32_t res, const float* atab, float act_scale, int relu) {
    const float2 rf = unpack_f16x2(res);
    float r0 = d0 + bias[0] + rf.x, r1 = d1 + bias[1] + rf.y;
    if (atab) { r0 = fmaf(act_scale, atab[0], r0); r1 = fmaf(act_scale, atab[1], r1); }
    if (relu) { r0 = fmaxf(r0, 0.0f); r1 = fmaxf(r1, 0.0f); }
    return pack_f16x2(r0, r1);
}
}  // namespace

// activation buffers hold fp16 (the host side types them float*: 2048 float slots per board)
MZ_DEVINL const __half* tower_board(const TowerArgs& a, int buf, int g) {
    const __half* base = reinterpret_cast<const __half*>(a.buf[buf]);
    if (buf == 0 && a.gather_parent)
        return base + ((size_t)g * a.pool_stride + a.gather_parent[g]) * (size_t)kBoardHalves;
    return base + (size_t)g * kBoardHalves;
}

__global__ void __launch_bounds__(kThreads, 1) conv_tower_tc_kernel(const __grid_constant__ TowerArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s_base = smem_u32(smem);
    const uint32_t s_w = s_base + Smem::w, s_a = s_base + Smem::a;
    float* s_bias = reinterpret_cast<float*>(smem + Smem::bias);
    const uint32_t bars = s_base + Smem::bars;
    // weight set = layer & 1
    auto bar_w_full = [&](int set, int tap) { return bars + 8u * (set * 9 + tap); };          // weights of (layer, tap) landed
    auto bar_w_empty = [&](int set, int tap) { return bars + 8u * (18 + set * 9 + tap); };    // last MMA of the layer on this tap done
    auto bar_a_full = [&](int s) { return bars + 8u * (36 + s); };
    auto bar_a_empty = [&](int s) { return bars + 8u * (38 + s); };
    auto bar_tile_done = [&](int k) { return bars + 8u * (44 + k); };      // layer output of my k-th tile stored
    auto bar_out_full = [&](int st) { return bars + 8u * (52 + st); };     // output tile staged in shared memory
    auto bar_out_empty = [&](int st) { return bars + 8u * (54 + st); };    // ... and drained by the bulk store

    const int n_tiles = (a.n + kBoards - 1) / kBoards;
    const int my_tiles = ((int)blockIdx.x < n_tiles) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int L = a.n_layers;

    // ---- one-time setup
    // zero the halo rows (the board rows are always overwritten by the bulk copies)
    for (int i = threadIdx.x; i < kStages * 2 * kHalo * (kRowBytes / 16); i += kThreads) {
        const int chunk = i % (kRowBytes / 16), r = (i / (kRowBytes / 16)) % (2 * kHalo), st = i / ((kRowBytes / 16) * 2 * kHalo);
        const int row = r < kHalo ? r : kRows - 2 * kHalo + r;
        reinterpret_cast<uint4*>(smem + Smem::a + st * kStageBytes + row * kRowBytes)[chunk] = make_uint4(0, 0, 0, 0);
    }
    for (int i = threadIdx.x; i < L * kC; i += kThreads) {
        const float* b = a.layer[i / kC].bias;
        s_bias[i] = b ? b[i % kC] : 0.0f;
    }
    if (threadIdx.x == 0) {
        for (int t = 0; t < 18; ++t) { mbar_init(bar_w_full(t / 9, t % 9), 1); mbar_init(bar_w_empty(t / 9, t % 9), kConsumerWarps); }
        for (int s = 0; s < kStages; ++s) {
            mbar_init(bar_a_full(s), 1);
            mbar_init(bar_a_empty(s), kConsumerWarps);   // one arrival per consumer warp
        }
        for (int k = 0; k < kTowerMaxTiles; ++k) mbar_init(bar_tile_done(k), 1);
        for (int st = 0; st < 2; ++st) { mbar_init(bar_out_full(st), kConsumerWarps); mbar_init(bar_out_empty(st), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic zero-fill -> async proxy readers
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp == kConsumerWarps) {
        // ================= producer =================
        int it = 0;
        // weights: two sets of nine tap slots; layer l uses set l & 1 and is loaded one layer ahead, as soon as the
        // last tile of layer l-2 has multiplied with the slot (so a layer never starts by waiting for its weights)
        auto load_weights = [&](int l) {
            const int set = l & 1, use = l >> 1;
            if (use > 0) mbar_wait(bar_w_empty(set, lane), (uint32_t)((use - 1) & 1));
            mbar_expect_tx(bar_w_full(set, lane), kTapBytes);
            bulk_g2s(s_w + set * kWBytes + lane * kTapBytes,
                     reinterpret_cast<const unsigned char*>(a.layer[l].w) + (size_t)lane * kTapBytes, kTapBytes, bar_w_full(set, lane));
        };
        if (my_tiles > 0 && lane < 9) { load_weights(0); if (L > 1) load_weights(1); }
        for (int l = 0; l < L; ++l) {
            if (l >= 1 && l + 1 < L && my_tiles > 0 && lane < 9) load_weights(l + 1);
            __syncwarp();
            const int in_buf = a.layer[l].in_buf;
            for (int k = 0; k < my_tiles; ++k, ++it) {
                const int tile = blockIdx.x + k * gridDim.x;
                const int s = it % kStages;
                const uint32_t ph = (it / kStages) & 1;
                if (lane == 0) {
                    mbar_wait(bar_a_empty(s), ph ^ 1);
                    if (l > 0) {
                        // this tile's input was written by this CTA's epilogue in the previous layer
                        mbar_wait(bar_tile_done(k), (uint32_t)((l - 1) & 1));
                        asm volatile("fence.proxy.async;" ::: "memory");
                    }
                }
                __syncwarp();
                const int nb = min(kBoards, a.n - tile * kBoards);
                if (a.debug_skip & 2) { if (lane == 0) mbar_arrive(bar_a_full(s)); __syncwarp(); continue; }
                if (lane == 0) mbar_expect_tx(bar_a_full(s), (uint32_t)nb * kPos * kRowBytes);
                __syncwarp();
                if (lane < nb) {                                           // one 8 KB bulk copy per board
                    const __half* src = tower_board(a, in_buf, tile * kBoards + lane);
                    bulk_g2s(s_a + s * kStageBytes + (kHalo + lane * kPos) * kRowBytes, src, kPos * kRowBytes, bar_a_full(s));
                }
            }
        }
    } else if (warp < kConsumerWarps) {
        // ================= MMA + epilogue: warpgroup wg owns board wg of every tile =================
        const int wg = warp >> 2;
        const int r0 = 16 * (warp & 3) + (lane >> 2);  // this thread's accumulator rows (board positions): r0, r0 + 8
        const int cq = 2 * (lane & 3);                 // ... and channels 8 j + cq, 8 j + cq + 1
        const int sw = lane >> 2;                      // r0 % 8 = (r0 + 8) % 8: chunk c of the row is stored at chunk c ^ sw
        int it = 0;
        for (int l = 0; l < L; ++l) {
            const TowerLayer& ly = a.layer[l];
            const float* bias = s_bias + l * kC;
            for (int k = 0; k < my_tiles; ++k, ++it) {
                const int tile = blockIdx.x + k * gridDim.x;
                const int s = it % kStages;
                const uint32_t ph = (it / kStages) & 1;
                const int g = tile * kBoards + wg;
                // ---- prefetch everything that does not depend on the accumulator
                uint32_t res[2][8];                     // residual, fp16x2 per (row, channel group)
                float act_scale = 0.0f;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int j = 0; j < 8; ++j) res[h][j] = 0u;
                if (g < a.n) {
                    if (ly.res_buf >= 0 && !(a.debug_skip & 8)) {
                        const __half* rp = tower_board(a, ly.res_buf, g);
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int j = 0; j < 8; ++j)        // written by bulk stores: not through L1
                                res[h][j] = __ldcg(reinterpret_cast<const unsigned int*>(rp + (size_t)(r0 + 8 * h) * kC + ((j ^ sw) << 3) + cq));
                    }
                    if (ly.action_table) act_scale = __fdiv_rn((float)a.action[g], (float)a.A);
                }
                mbar_wait(bar_a_full(s), ph);
                float d[32];
                if (a.debug_skip & 1) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) d[i] = 0.0f;
                    if (k == 0) for (int tap = 0; tap < 9; ++tap) mbar_wait(bar_w_full(l & 1, tap), (uint32_t)((l >> 1) & 1));
                } else {
                    const uint32_t a16 = ((s_a + s * kStageBytes + (kHalo + wg * kPos) * kRowBytes) >> 4) | kDescLoFlags;
                    const uint32_t w16 = ((s_w + (uint32_t)((l & 1) * kWBytes)) >> 4) | kDescLoFlags;
                    board_conv(d, a16, w16, bar_w_full(l & 1, 0), k == 0, (uint32_t)((l >> 1) & 1));
                }
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(bar_a_empty(s));                   // smem stage reusable: this warp's MMAs have read it
                    if (k == my_tiles - 1)
                        for (int tap = 0; tap < 9; ++tap) mbar_arrive(bar_w_empty(l & 1, tap));   // slot reusable by layer l + 2
                }
                // the output tile is staged in shared memory in the global board layout and leaves with one bulk store
                // per board (store warp): the epilogue never waits for global memory
                const int st = it & 1;
                mbar_wait(bar_out_empty(st), ((uint32_t)(it >> 1) & 1u) ^ 1u);
                if (g < a.n) {
                    unsigned char* dst = smem + Smem::out + st * kOutBytes + wg * kPos * kRowBytes;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int p = r0 + 8 * h;
                        const int y = p / 8 - 1, x = p % 8;
                        const bool inside = (y >= 0 && y < a.H && x < a.W);
                        const float* atab = ly.action_table ? ly.action_table + (size_t)p * kC + cq : nullptr;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const uint32_t o = inside ? finish_pair(d[4 * j + 2 * h], d[4 * j + 2 * h + 1], bias + 8 * j + cq, res[h][j],
                                                                    atab ? atab + 8 * j : nullptr, act_scale, ly.relu)
                                                      : 0u;
                            *reinterpret_cast<uint32_t*>(dst + p * kRowBytes + ((j ^ sw) << 4) + 2 * cq) = o;
                        }
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic smem writes -> bulk-copy reader
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_out_full(st));
            }
        }
    } else {
        // ================= output store =================
        if (lane == 0) {
            int it = 0;
            for (int l = 0; l < L; ++l) {
                __half* out = reinterpret_cast<__half*>(a.buf[a.layer[l].out_buf]);
                for (int k = 0; k < my_tiles; ++k, ++it) {
                    const int st = it & 1;
                    const int tile = blockIdx.x + k * gridDim.x;
                    const int nb = min(kBoards, a.n - tile * kBoards);
                    mbar_wait(bar_out_full(st), (uint32_t)(it >> 1) & 1u);
                    if (!(a.debug_skip & 4)) {
                        for (int b = 0; b < nb; ++b)
                            bulk_s2g(out + (size_t)(tile * kBoards + b) * kBoardHalves,
                                     s_base + Smem::out + st * kOutBytes + b * (kPos * kRowBytes), kPos * kRowBytes);
                    }
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    // the staging buffer is free as soon as the copy engine has READ it; the tile counts as stored
                    // (next layer may load it) only when the writes are complete - tracked one store behind, so two
                    // stores are in flight inside a layer, and drained at the end of every layer
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    mbar_arrive(bar_out_empty(st));
                    if (k > 0) {
                        asm volatile("cp.async.bulk.wait_group 1;" ::: "memory");
                        if (l + 1 < L) { __threadfence(); mbar_arrive(bar_tile_done(k - 1)); }
                    }
                    if (k == my_tiles - 1) {
                        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
                        if (l + 1 < L) { __threadfence(); mbar_arrive(bar_tile_done(k)); }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Resident tower: the same convolutions, but the activations of a CTA's tiles never leave shared memory between the
// layers.  Two activation buffers B0 / B1 hold the CTA's (up to kResTiles) tiles back to back in the board layout
// (consecutive boards are separated by their own zero padding rows, so a tap window of a real position never leaves
// its board); layer l reads B[l & 1] and writes B[(l & 1) ^ 1]; the second conv of a block adds the residual IN PLACE
// (the block input is what the output buffer still holds, and a row is read and overwritten by the same thread).
// Global memory is touched three times per tower: bulk loads of the input boards, the weight taps (one slot set,
// refilled for layer l+1 while the last tile of layer l multiplies), bulk stores of the last layer's boards.  A
// warpgroup only ever reads the rows of its own boards for the positions it keeps (other boards' rows only enter
// padding outputs, which are stored as zeros), so the two warpgroups never wait for each other: a warpgroup's own
// MMA -> epilogue -> next MMA order covers every hazard.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kResTiles = 4;
constexpr int kResRows = kResTiles * kBoards * kPos + 2 * kHalo;      // 544
constexpr int kResBufBytes = kResRows * kRowBytes;                    // 69632 (multiple of 1024: swizzle phase kept)

struct SmemR {
    static constexpr int w = 0;
    static constexpr int act = kWBytes;                                    // B0 | B1
    static constexpr int bias = act + 2 * kResBufBytes;
    static constexpr int bars = bias + kTowerMaxLayers * kC * 4;
    static constexpr int total = bars + 32 * 8;
};
static_assert(SmemR::total <= 232448, "shared memory budget");
static_assert(SmemR::act % 1024 == 0 && kResBufBytes % 1024 == 0, "activation buffers must keep the 1024-byte swizzle phase");

__global__ void __launch_bounds__(kThreadsR, 1) conv_tower_resident_kernel(const __grid_constant__ TowerArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s_base = smem_u32(smem);
    const uint32_t s_w = s_base + SmemR::w, s_act = s_base + SmemR::act;
    float* s_bias = reinterpret_cast<float*>(smem + SmemR::bias);
    const uint32_t bars = s_base + SmemR::bars;
    auto bar_w_full = [&](int tap) { return bars + 8u * tap; };
    auto bar_w_empty = [&](int tap) { return bars + 8u * (9 + tap); };
    auto bar_in_full = [&](int k) { return bars + 8u * (18 + k); };         // input boards of my k-th tile landed

    const int n_tiles = (a.n + kBoards - 1) / kBoards;
    const int my_tiles = ((int)blockIdx.x < n_tiles) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int L = a.n_layers;

    // ---- one-time setup: zero halos of both buffers, biases, barriers
    for (int i = threadIdx.x; i < 2 * 2 * kHalo * (kRowBytes / 16); i += kThreadsR) {
        const int chunk = i % (kRowBytes / 16), r = (i / (kRowBytes / 16)) % (2 * kHalo), bf = i / ((kRowBytes / 16) * 2 * kHalo);
        const int row = r < kHalo ? r : kResRows - 2 * kHalo + r;
        reinterpret_cast<uint4*>(smem + SmemR::act + bf * kResBufBytes + row * kRowBytes)[chunk] = make_uint4(0, 0, 0, 0);
    }
    for (int i = threadIdx.x; i < L * kC; i += kThreadsR) {
        const float* b = a.layer[i / kC].bias;
        s_bias[i] = b ? b[i % kC] : 0.0f;
    }
    if (threadIdx.x == 0) {
        for (int t = 0; t < 9; ++t) { mbar_init(bar_w_full(t), 1); mbar_init(bar_w_empty(t), kConsumerWarps); }
        for (int k = 0; k < kResTiles; ++k) mbar_init(bar_in_full(k), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ================= producer: weights of every layer, input boards once =================
        pdl_launch_dependents();
        if (my_tiles > 0 && lane < 9) {
            mbar_expect_tx(bar_w_full(lane), kTapBytes);
            bulk_g2s(s_w + lane * kTapBytes, reinterpret_cast<const unsigned char*>(a.layer[0].w) + (size_t)lane * kTapBytes, kTapBytes,
                     bar_w_full(lane));
        }
        pdl_wait();                                    // weights are constants; the boards come from the previous kernel
        __syncwarp();
        const int in_buf = a.layer[0].in_buf;
        for (int k = 0; k < my_tiles; ++k) {
            const int tile = blockIdx.x + k * gridDim.x;
            const int nb = min(kBoards, a.n - tile * kBoards);
            if (lane == 0) mbar_expect_tx(bar_in_full(k), (uint32_t)nb * kPos * kRowBytes);
            __syncwarp();
            if (lane < nb)
                bulk_g2s(s_act + (kHalo + (k * kBoards + lane) * kPos) * kRowBytes, tower_board(a, in_buf, tile * kBoards + lane),
                         kPos * kRowBytes, bar_in_full(k));
        }
        for (int l = 1; l < L; ++l) {
            if (my_tiles > 0 && lane < 9) {
                mbar_wait(bar_w_empty(lane), (uint32_t)((l - 1) & 1));        // last tile of layer l-1 is done with this tap
                mbar_expect_tx(bar_w_full(lane), kTapBytes);
                bulk_g2s(s_w + lane * kTapBytes, reinterpret_cast<const unsigned char*>(a.layer[l].w) + (size_t)lane * kTapBytes,
                         kTapBytes, bar_w_full(lane));
            }
            __syncwarp();
        }
    } else {
        // ================= MMA + epilogue: warpgroup wg owns board wg of every tile =================
        pdl_wait();                                    // reads a.action (written by the tree kernel)
        const int wg = warp >> 2;
        const int r0 = 16 * (warp & 3) + (lane >> 2);  // accumulator rows r0, r0 + 8; channels 8 j + cq (+1)
        const int cq = 2 * (lane & 3);
        const int sw = lane >> 2;                      // chunk c of the row is stored at chunk c ^ sw
        const bool store_lead = (threadIdx.x & 127) == 0;
        for (int l = 0; l < L; ++l) {
            const TowerLayer& ly = a.layer[l];
            const float* bias = s_bias + l * kC;
            const bool last = l == L - 1;
            for (int k = 0; k < my_tiles; ++k) {
                const int tile = blockIdx.x + k * gridDim.x;
                const int g = tile * kBoards + wg;
                const int brow = kHalo + (k * kBoards + wg) * kPos;               // row 0 of my board in a buffer
                float act_scale = 0.0f;
                if (g < a.n && ly.action_table) act_scale = __fdiv_rn((float)a.action[g], (float)a.A);
                if (l == 0) mbar_wait(bar_in_full(k), 0);
                float d[32];
                if (a.debug_skip & 1) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) d[i] = 0.0f;
                    if (k == 0) for (int tap = 0; tap < 9; ++tap) mbar_wait(bar_w_full(tap), (uint32_t)(l & 1));
                } else {
                    const uint32_t a16 = ((s_act + (uint32_t)((l & 1) * kResBufBytes + brow * kRowBytes)) >> 4) | kDescLoFlags;
                    board_conv(d, a16, (s_w >> 4) | kDescLoFlags, bar_w_full(0), k == 0, (uint32_t)(l & 1));
                }
                __syncwarp();
                if (lane == 0 && k == my_tiles - 1)
                    for (int tap = 0; tap < 9; ++tap) mbar_arrive(bar_w_empty(tap));
                unsigned char* ob = smem + SmemR::act + ((l & 1) ^ 1) * kResBufBytes + brow * kRowBytes;   // output board
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int p = r0 + 8 * h;
                    const int y = p / 8 - 1, x = p % 8;
                    const bool live = (y >= 0 && y < a.H && x < a.W) && g < a.n;
                    const float* atab = ly.action_table ? ly.action_table + (size_t)p * kC + cq : nullptr;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        uint32_t* slot = reinterpret_cast<uint32_t*>(ob + p * kRowBytes + ((j ^ sw) << 4) + 2 * cq);
                        uint32_t o = 0u;                                   // zeros on padding rows and missing boards
                        if (live)
                            o = finish_pair(d[4 * j + 2 * h], d[4 * j + 2 * h + 1], bias + 8 * j + cq, ly.res_buf >= 0 ? *slot : 0u,
                                            atab ? atab + 8 * j : nullptr, act_scale, ly.relu);   // residual: the block input, in place
                        *slot = o;
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic smem writes -> wgmma / bulk-copy readers
                warpgroup_sync(wg);
                if (last && store_lead && g < a.n && !(a.debug_skip & 4)) {
                    bulk_s2g(reinterpret_cast<__half*>(a.buf[ly.out_buf]) + (size_t)g * kBoardHalves, smem_u32(ob), kPos * kRowBytes);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (store_lead) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// the resident kernel needs the block structure: every residual is the input of the layer before, buffers alternate
static bool tower_is_resident_shape(const TowerArgs& a, int tiles_per_cta) {
    if (a.n_layers < 2 || tiles_per_cta > kResTiles) return false;
    for (int l = 0; l < a.n_layers; ++l) {
        const TowerLayer& t = a.layer[l];
        if (l > 0 && t.in_buf != a.layer[l - 1].out_buf) return false;
        if (t.res_buf >= 0 && (l == 0 || t.res_buf != a.layer[l - 1].in_buf)) return false;
    }
    return true;
}

static int tower_ctas_per_sm() {
    static int per_sm = 0;
    if (per_sm == 0) {
        int occ = 1;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, conv_tower_tc_kernel, kThreads, Smem::total) != cudaSuccess || occ < 1) occ = 1;
        if (getenv("MZ_TC_VERBOSE")) fprintf(stderr, "[conv_tower_tc] occupancy %d CTAs/SM, %d B shared per CTA\n", occ, Smem::total);
        const char* e = getenv("MZ_TC_CTAS");           // A/B switch: force one CTA per SM
        if (e && atoi(e) >= 1 && atoi(e) < occ) occ = atoi(e);
        per_sm = occ > 2 ? 2 : occ;
    }
    return per_sm;
}

cudaError_t launch_conv_tower_tc(const TowerArgs& a, int sm_count, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(conv_tower_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Smem::total);
        if (e != cudaSuccess) return e;
        // all of the SM's unified L1/shared array as shared memory, so two CTAs fit side by side
        e = cudaFuncSetAttribute(conv_tower_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    if (a.n_layers < 1 || a.n_layers > kTowerMaxLayers) return cudaErrorInvalidValue;
    const int n_tiles = (a.n + kBoards - 1) / kBoards;
    // up to two co-resident CTAs per SM where shared memory allows (the occupancy query decides)
    const int slots = sm_count * tower_ctas_per_sm();
    const int grid = n_tiles < slots ? n_tiles : slots;
    if (a.n_layers > 1 && (n_tiles + grid - 1) / grid > kTowerMaxTiles) return cudaErrorInvalidConfiguration;
    const char* nr = getenv("MZ_TC_NO_RESIDENT");            // A/B switch (tests compare both kernels)
    const bool no_resident = nr && nr[0] == '1';
    if (!no_resident && tower_is_resident_shape(a, (n_tiles + sm_count - 1) / sm_count)) {
        static bool attr_r = false;
        if (!attr_r) {
            cudaError_t e = cudaFuncSetAttribute(conv_tower_resident_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemR::total);
            if (e != cudaSuccess) return e;
            attr_r = true;
        }
        const int grid_r = n_tiles < sm_count ? n_tiles : sm_count;
        cudaError_t e = launch_chained(conv_tower_resident_kernel, dim3(grid_r), dim3(kThreadsR), SmemR::total, stream, a);
        return e != cudaSuccess ? e : cudaGetLastError();
    }
    cudaError_t e = launch_chained(conv_tower_tc_kernel, dim3(grid), dim3(kThreads), Smem::total, stream, a);
    return e != cudaSuccess ? e : cudaGetLastError();
}

int conv_tc_max_boards_fused(int sm_count) { return sm_count * kTowerMaxTiles * kBoards; }   // conservative: one CTA per SM

bool conv_tc_supported(int C, int H, int W) { return C == kC && H >= 1 && H <= 6 && W >= 1 && W <= 7; }
int conv_tc_board_elems(bool split) { return split ? kBoardHalves : kBoardHalves / 2; }      // float slots per board (fp16 plane, or x_h | x_l planes)

}  // namespace mz
