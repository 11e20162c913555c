// 256-channel residual towers on the tensor cores at fp32-grade accuracy (games/atari.py's 16 x 256 net on its 6 x 6 hidden
// board), opt-in with MZ_TC_WIDE=3 on the dense fp32 route of resnet_inference.
//
// Numerics, padding and the range guard are conv_wide.cu's, unchanged: split fp16 operands x = x_h + x_l/2^11, w = (w_h +
// w_l)/s with s a power of two per output channel, three wgmma partial products per K-step (x_l w_l dropped), fp32
// accumulation, an epilogue that forms acc + acc_l/2^11, unscales, adds the bias, the fp32 residual and the action-plane
// term and applies the ReLU; padding positions are stored as zeros; activations beyond the fp16 range bump sat_count.
//
// Split N across a CTA pair, stack boards in M.  One cluster of two CTAs runs a group of `boards` boards.  CTA rank r
// computes output channels [128 r, 128 r + 128) over the full K of 256 input channels:
//   - each CTA holds all 256 input channels of its boards: 4 K-quarters of 64 channels, x_h and x_l, so 8 swizzled planes;
//   - each CTA streams only its own N-half of the weights: one ring stage is one tap x one K-quarter x 128 output channels
//     (w_h | w_l, the 32 KB stage of conv_wide.cu), 36 stages per layer (9 taps x 4 K-quarters);
//   - per stage each warpgroup issues 4 K-steps x 2 N-halves x 3 m64n64k16, and keeps dm[2][32], dl[2][32] (128 registers).
//
// Board rows: with row stride S = W + 1, position (y, x) of board b is plane row 1 + S + b (H + 1) S + y S + x.  Column W of
// every row is zero (the right pad of row y, the left pad of row y + 1); the S rows between two boards are the bottom pad
// of one board and the top pad of the next; row 0 is the guard and rows 1 .. S the top pad of board 0.  A tap (dy, dx)
// moves the A descriptor by dy S + dx rows.  The interior (B (H + 1) - 1) S rows are cut into 64-row M-tiles, one warpgroup
// each; the separator rows and the zero columns are computed and stored as zero, rows past the interior are masked, and an
// empty board slot (the last group of an odd batch) is stored as zero like a separator.
//
// Shared memory (Atari's 6 x 6, S = 7, 2 boards per CTA: 91 interior rows, 2 M-tiles, 256 threads):
//   activations   8 planes (x_h, x_l) x 4 K-quarters x 112 rows (1 + 7 + 2 x 49 = 106, rounded to 8) x 128 B  114,688 B
//   weight ring   2 stages x 32 KB                                                                          65,536 B
//   residual      fp32, 91 interior rows x 136 floats (the CTA's 128 channels + 8 against bank conflicts)    49,504 B
//   barriers                                                                                                    32 B
//   total 229,760 B of the 232,448 B a CTA may take.  Three boards need 3 M-tiles and do not fit; one board fits up to
//   9 x 9.  Registers: the accumulators take 128 of the 255 that __launch_bounds__(256, 1) leaves (tests read the SASS).
// Weight traffic: each CTA pulls its 36 x 32 KB = 1.18 MB per layer from L2 for `boards` boards.
//
// Exchange through distributed shared memory.  Each CTA's epilogue stores its 128 output channels (2 K-quarters) into its
// own planes and into the peer's, at the same plane rows (so the same 128B-swizzle phase).  Ordering, per layer l:
//   1. wgmma.wait_group 0, then a cluster barrier (arrive.release / wait.acquire): every MMA of layer l in BOTH CTAs has
//      read the planes before either epilogue rewrites a K-quarter the other CTA's MMAs read;
//   2. the epilogue writes its K-quarters locally (generic proxy) and remotely (generic proxy, st.shared::cluster);
//   3. fence.proxy.async.shared::cluster by every writer, then a cluster barrier: the generic writes of both CTAs, local
//      and remote, are ordered before any wgmma (async proxy) of layer l + 1 reads them.
// The first remote store follows the barrier of step 1 of layer 0, which the peer reaches only after zeroing and filling
// its planes; the barrier of step 3 after the last layer keeps each CTA resident until its peer has stopped writing into
// it.  Each CTA keeps the fp32 residual of its own 128 channels and writes those channels of the NCHW fp32 output.
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

#include "conv_wide.h"
#include "launch.h"
#include "tc_common.cuh"

namespace mz {

namespace {

using namespace tc;

constexpr int kC = kWide256C;
constexpr int kHalf = 128;                            // output channels per CTA of the pair
constexpr int kRowBytes = 128;                        // one 64-channel K-quarter of a position, fp16
constexpr int kStageBytes = 256 * kRowBytes;          // 32768: [w_h cout 0..127 | w_l cout 0..127][64 cin] of one N-half
constexpr int kKParts = kC / 64;                      // 4 K-quarters
constexpr int kStagesPerLayer = 9 * kKParts;          // 36
constexpr int kRingStages = 2;
constexpr int kResStride = kHalf + 8;
constexpr int kMaxMTiles = 2;
constexpr int kMaxBoards = 8;                         // boards stacked per CTA pair at most (1 x 1 boards)
constexpr int kMaxThreads = 128 * kMaxMTiles;
constexpr int kRegCap = 255;                          // __launch_bounds__(256, 1)
constexpr int kSmemLimit = 232448;
constexpr float kLoScale = 2048.0f, kLoUnscale = 1.0f / 2048.0f;

}  // namespace

// launched in clusters of two CTAs (launch_chained_cluster), grid 2 ceil(n / boards): cluster k runs boards
// g0 + k boards .. g0 + (k + 1) boards - 1 (those below g0 + n)
__global__ void __launch_bounds__(kMaxThreads, 1) conv_tower_wide256_kernel(const __grid_constant__ Wide256Args a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const int S = a.S, W = a.W, H = a.H, HW = H * W, BS = (H + 1) * S, B = a.boards;
    const uint32_t plane = (uint32_t)a.plane_bytes;
    const uint32_t s_base = smem_u32(smem);
    const uint32_t s_ring = s_base + 2 * kKParts * plane;
    float* res = reinterpret_cast<float*>(smem + a.res_off);
    const uint32_t bars = s_base + (uint32_t)a.bar_off;
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (kRingStages + s); };
    const int L = a.n_layers, total = L * kStagesPerLayer;
    const int first = (int)(blockIdx.x >> 1) * B;      // the group's first board, relative to g0
    const int n_real = min(B, a.n - first);             // real boards of the group (the rest are empty slots)
    const int rank = (int)cluster_rank();

    if (threadIdx.x == 0) {
        for (int s = 0; s < kRingStages; ++s) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), blockDim.x >> 5); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (uint32_t i = threadIdx.x; i < 2 * kKParts * plane / 16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    auto load_stage = [&](int q) {                     // thread 0: stage q of my N-half into ring slot q % 2
        const int s = q & 1;
        mbar_expect_tx(bar_full(s), kStageBytes);
        bulk_g2s(s_ring + s * kStageBytes,
                 reinterpret_cast<const unsigned char*>(a.layer[q / kStagesPerLayer].w) +
                     (size_t)(rank * kStagesPerLayer + q % kStagesPerLayer) * kStageBytes,
                 kStageBytes, bar_full(s));
    };
    if (threadIdx.x == 0) {
        pdl_launch_dependents();
        load_stage(0);                                 // weights are constants; the boards come from the previous kernel
        load_stage(1);
    }
    pdl_wait();

    // ---- the boards: NCHW fp32 -> x_h / x_l planes of all 256 channels; the first block's residual of my 128 channels
    const bool res_in = !a.stem;
    float peak = 0.0f;                                 // largest |activation| this thread read or stored
    const int per_board = kC * HW;
    for (int i = threadIdx.x; i < n_real * per_board; i += blockDim.x) {
        const int b = i / per_board, e = i - b * per_board, c = e / HW, p = e - c * HW, y = p / W, x = p - y * W;
        const int g = a.g0 + first + b;
        const size_t slot = a.gather_parent ? (size_t)g * a.pool_stride + a.gather_parent[g] : (size_t)g;
        const float v = __ldg(a.in + slot * (size_t)per_board + e);
        peak = fmaxf(peak, fabsf(v));
        const int ir = b * BS + y * S + x;             // interior row
        const int row = 1 + S + ir;
        const uint32_t off = (uint32_t)(row * kRowBytes + ((((c & 63) >> 3) ^ (row & 7)) << 4) + (c & 7) * 2);
        split_store(smem + (c >> 6) * plane + off, smem + (kKParts + (c >> 6)) * plane + off, v);
        if (res_in && (c >> 7) == rank) res[ir * kResStride + (c & 127)] = v;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic smem writes -> wgmma readers
    __syncthreads();

    const int r0 = 16 * (warp & 3) + (lane >> 2);      // accumulator rows r0, r0 + 8 of my M-tile; channels 8 j + cq (+1)
    const int cq = 2 * (lane & 3);
    const int i0 = 64 * wg + r0;                       // interior row of accumulator row r0
    const uint32_t plane16 = plane >> 4;
    const uint32_t a16 = ((s_base + (uint32_t)((1 + S + 64 * wg) * kRowBytes)) >> 4) | kDescLoFlags;   // my M-tile, plane 0
    const uint32_t ring16 = (s_ring >> 4) | kDescLoFlags;
    float dm[2][32], dl[2][32];                        // x_h (w_h + w_l) | x_l w_h, for the two 64-channel halves of my N
    auto release = [&](int p) {                        // stage p's MMAs of this warp are complete
        if (lane == 0) mbar_arrive(bar_empty(p & 1));
        if (threadIdx.x == 0 && p + kRingStages < total) {
            mbar_wait(bar_empty(p & 1), (uint32_t)((p >> 1) & 1));
            load_stage(p + kRingStages);
        }
        __syncwarp();
    };
    int q = 0;
    for (int l = 0; l < L; ++l) {
        const WideLayer& ly = a.layer[l];
        wgmma_fence();
#pragma unroll 1
        for (int t = 0; t < kStagesPerLayer; ++t, ++q) {
            const int tap = t >> 2, kq = t & 3;
            mbar_wait(bar_full(q & 1), (uint32_t)((q >> 1) & 1));
            const int shift = (tap / 3 - 1) * S + (tap % 3 - 1);
            const uint32_t ah = a16 + (uint32_t)kq * plane16 + (uint32_t)(shift * (kRowBytes / 16));
            const uint32_t al = ah + kKParts * plane16;
            const uint32_t b16 = ring16 + (uint32_t)((q & 1) * (kStageBytes / 16));
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
                for (int nh = 0; nh < 2; ++nh) {
                    const uint32_t bh = b16 + (uint32_t)(nh * (64 * kRowBytes / 16) + ks * 2);     // w_h rows; w_l 128 further
                    const uint32_t acc = (t | ks) != 0;
                    wgmma_m64n64k16(dm[nh], ah + ks * 2, bh, acc);
                    wgmma_m64n64k16(dm[nh], ah + ks * 2, bh + (uint32_t)(128 * kRowBytes / 16), 1);
                    wgmma_m64n64k16(dl[nh], al + ks * 2, bh, acc);
                }
            }
            wgmma_commit();
            if (t > 0) {
                wgmma_wait_one();
                release(q - 1);
            }
        }
        wgmma_wait_all();
        release(q - 1);
        cluster_barrier();                             // every M-tile's MMAs of layer l in both CTAs are complete

        const int bl = l - a.stem;                     // conv index inside the blocks (-1: the stem)
        const bool add_res = bl >= 0 && (bl & 1);
        const bool keep = l + 1 < L && (bl < 0 || (bl & 1));       // this output is the input of a block
        const bool last = l == L - 1;
        const int me = (int)cluster_rank();            // (asked again: the MMA loop's accumulators fill the registers)
        const uint32_t peer_base = map_to_cta(s_base, (uint32_t)(me ^ 1));
        const float* table = ly.action_table;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = i0 + 8 * h;
            if (i >= a.interior) continue;             // masked rows
            const int b = i / BS, yb = i - b * BS, y = yb / S, x = yb - y * S;
            const bool live = x < W && y < H && first + b < a.n;      // not a zero column, separator row or empty slot
            const int row = 1 + S + i;
            const int g = a.g0 + first + b;
            const float act_scale = table && live ? __fdiv_rn((float)a.action[g], (float)a.A) : 0.0f;
            float* dst = a.out + (size_t)g * kC * HW;
#pragma unroll
            for (int nh = 0; nh < 2; ++nh)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int cl = 64 * nh + 8 * j + cq, c = kHalf * me + cl;
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int k = 4 * j + 2 * h + e;
                        float u = fmaf(dl[nh][k], kLoUnscale, dm[nh][k]) * __ldg(ly.scale + c + e) + (ly.bias ? __ldg(ly.bias + c + e) : 0.0f);
                        if (add_res) u += res[i * kResStride + cl + e];
                        if (table && live) u = fmaf(act_scale, __ldg(table + (size_t)(y * W + x) * kC + c + e), u);
                        u = fmaxf(u, 0.0f);
                        if (!live) u = 0.0f;           // zero columns, separator rows and empty slots stay zero
                        peak = fmaxf(peak, fabsf(u));
                        v[e] = u;
                    }
                    if (keep) *reinterpret_cast<float2*>(res + i * kResStride + cl) = make_float2(v[0], v[1]);
                    if (last) {
                        if (live) {
                            dst[(size_t)c * HW + y * W + x] = v[0];
                            dst[(size_t)(c + 1) * HW + y * W + x] = v[1];
                        }
                    } else {
                        const uint32_t off = (uint32_t)(row * kRowBytes + ((j ^ (row & 7)) << 4) + 2 * cq);
                        const uint32_t hw = pack_f16x2(v[0], v[1]);
                        const float2 hf = unpack_f16x2(hw);
                        const uint32_t lw = pack_f16x2((v[0] - hf.x) * kLoScale, (v[1] - hf.y) * kLoScale);
                        const uint32_t ph = (uint32_t)(2 * me + nh) * plane + off, pl = ph + kKParts * plane;
                        *reinterpret_cast<uint32_t*>(smem + ph) = hw;
                        *reinterpret_cast<uint32_t*>(smem + pl) = lw;
                        st_cluster_u32(peer_base + ph, hw);      // the peer's copy of my K-quarter, same row and phase
                        st_cluster_u32(peer_base + pl, lw);
                    }
                }
        }
        asm volatile("fence.proxy.async.shared::cluster;" ::: "memory");      // local and remote writes -> both CTAs' wgmma
        cluster_barrier();                             // after the last layer: the peer no longer writes into my planes
    }
    if (peak > 65504.0f && a.sat_count) atomicAdd(a.sat_count, 1);
}

namespace {
enum Wide256Fit { kFits256, kTooManyMTiles256, kOverSmem256, kOverRing256 };

// Budget of one CTA holding `boards` stacked boards of H x W (all 256 input channels, 128 output channels)
Wide256Fit wide256_budget(int boards, int H, int W, int sm_count, int layers, Wide256Plan* p) {
    const int S = W + 1, interior = (boards * (H + 1) - 1) * S;
    const int m_tiles = (interior + 63) / 64;
    if (m_tiles > kMaxMTiles) return kTooManyMTiles256;
    const int rows = (1 + S + boards * (H + 1) * S + 7) & ~7;
    const size_t planes = (size_t)2 * kKParts * rows * kRowBytes;
    const size_t res = (size_t)interior * kResStride * 4;
    const size_t smem = planes + (size_t)kRingStages * kStageBytes + res + 8 * 2 * kRingStages;
    if (smem > (size_t)kSmemLimit) return kOverSmem256;
    // masked output rows read at most 2 S + 64 m_tiles + 1 rows from the last plane's start: they must stay inside the ring
    if ((2 * S + 64 * m_tiles + 1 - rows) * kRowBytes > kRingStages * kStageBytes) return kOverRing256;
    p->boards = boards;
    p->m_tiles = m_tiles;
    p->threads = 128 * m_tiles;
    p->rows = rows;
    p->interior = interior;
    p->stages = kRingStages;
    p->smem = smem;
    p->layers = layers;
    const int by_smem = (int)(233472 / (smem + 2048));           // 228 KB per SM; per CTA 1 KB reserved + 1 KB static (alignment)
    const int by_regs = 65536 / (p->threads * kRegCap);
    p->ctas_per_sm = std::min(std::min(by_smem, by_regs), 2048 / p->threads);
    p->wave = p->ctas_per_sm * sm_count / 2 * boards;  // boards per wave, as planned: the GPCs may hold fewer pairs
    p->launches = 1;                                   // one CTA pair per group of boards: any batch is one launch
    p->reg_cap = kRegCap;
    return kFits256;
}
}  // namespace

bool wide256_plan(int n, int C, int H, int W, int layers, int sm_count, int force_boards, Wide256Plan* p, const char** why) {
    *p = Wide256Plan{};
    if (C != kC) { *why = "the 256-channel towers take 256 channels"; return false; }
    if (n < 1 || H < 1 || W < 1 || sm_count < 1) { *why = "empty shape"; return false; }
    if (force_boards < 0 || force_boards > kMaxBoards) { *why = "forced boards per CTA pair: 0 (planned) or 1 to 8"; return false; }
    if (layers < 1 || layers > kWide256MaxLayers) { *why = "1 to 33 layers (a stem and up to 16 blocks)"; return false; }
    Wide256Fit fit = kTooManyMTiles256;
    // the largest number of stacked boards that fits (or the forced one)
    for (int b = force_boards ? force_boards : kMaxBoards; b >= (force_boards ? force_boards : 1); --b) {
        fit = wide256_budget(b, H, W, sm_count, layers, p);
        if (fit == kFits256) break;
    }
    switch (fit) {
        case kTooManyMTiles256:
            *why = force_boards > 1 ? "the forced boards per CTA exceed the 128 rows of two M-tiles"
                                    : "board too large: H x (W + 1) exceeds the 128 rows of two M-tiles";
            return false;
        case kOverSmem256:
            *why = force_boards > 1 ? "the forced boards per CTA exceed shared memory"
                                    : "board too large: activations, weight ring and residual exceed shared memory";
            return false;
        case kOverRing256: *why = "tap windows overrun the ring"; return false;
        case kFits256: break;
    }
    return true;
}

cudaError_t launch_wide256_tower(Wide256Args a, const Wide256Plan& p, cudaStream_t stream) {
    static size_t attr_smem = 0;
    if (attr_smem < p.smem) {
        cudaError_t e = cudaFuncSetAttribute(conv_tower_wide256_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
        if (e != cudaSuccess) return e;
        attr_smem = p.smem;
    }
    if (a.n_layers != p.layers || a.n < 1 || p.boards < 1) return cudaErrorInvalidValue;
    for (int l = 1; l < a.n_layers; ++l) if (a.layer[l].action_table) return cudaErrorInvalidValue;   // a table belongs to the stem
    if (a.layer[0].action_table && (!a.stem || !a.action)) return cudaErrorInvalidValue;
    a.S = a.W + 1;
    a.boards = p.boards;
    a.interior = p.interior;
    a.plane_bytes = p.rows * kRowBytes;
    a.res_off = 2 * kKParts * a.plane_bytes + kRingStages * kStageBytes;
    a.bar_off = a.res_off + p.interior * kResStride * 4;
    const int groups = (a.n + p.boards - 1) / p.boards;
    cudaError_t e = launch_chained_cluster(conv_tower_wide256_kernel, dim3(2 * groups), dim3(p.threads), dim3(2, 1, 1), p.smem,
                                           stream, a);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

}  // namespace mz
