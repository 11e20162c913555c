// 128-channel residual towers on the tensor cores at fp32-grade accuracy (Gomoku's 6 x 128 net on 11 x 11), opt-in with
// MZ_TC_WIDE=1 on the dense fp32 route of resnet_inference.
//
// Numerics: the x3 recipe of conv_x3.cu, unchanged.  x = x_h + x_l/2^11 (x_l the scaled fp16 remainder), w = (w_h + w_l)/s
// with s a power of two per output channel, three wgmma partial products per K-step (x_h w_h and x_h w_l into one
// accumulator, x_l w_h into a second; x_l w_l dropped), the epilogue forms acc + acc_l/2^11, unscales, adds the bias, the
// residual and the action-plane term and applies the ReLU.  Padding positions are stored as zeros.  The block residual is
// kept in fp32 (the tower input exactly as read, later layers as computed).  Activations beyond the fp16 range bump
// sat_count: the handle then leaves these towers for the fp32 CUDA-core ones (resnet.cu).
//
// Layout: dense in, dense out.  One CTA runs the whole tower of ONE board: it reads the NCHW fp32 board (a workspace, the
// rescaled-state scratch or a pool slot), splits it into swizzled fp16 planes in shared memory and writes NCHW fp32 after
// the last layer.  No other board layout leaves the kernel.
//
// Board rows: position (y, x) is plane row 1 + (y + 1) S + x with S = W + 1.  Column W of every row is zero and serves as
// the right pad of row y and the left pad of row y + 1; rows 1 .. S and the S rows after the board are zero, row 0 is the
// guard the top-left tap of position (0, 0) reads.  A tap (dy, dx) moves the A descriptor by dy S + dx rows (the 128B
// swizzle works on absolute address bits, as in conv_x3.cu).  The H S interior rows (board + zero columns) are cut into
// m_tiles = ceil(H S / 64) M-tiles, one warpgroup each; output rows past H S are masked (never stored) and the A rows they
// read may run past the plane into the next one or into the weight ring: wgmma rows are independent.
//
// Shared memory (11 x 11, S = 12, 132 interior rows, 3 M-tiles, 384 threads):
//   activations   4 planes (x_h, x_l) x (K-half 0, 1) x 160 rows x 128 B                      80 KB
//   weight ring   2 stages x (one tap x one 64-channel K-half: 256 rows w_h | w_l x 128 B)     64 KB
//   residual      fp32, 132 interior rows x 136 floats (128 channels + 8 against bank conflicts) 70 KB
//   barriers                                                                                    32 B
//   total 219,296 B of the 232,448 B a CTA may take.  12 x 12 would need 244,640 B and 15 x 15 five M-tiles: refused.
// Registers: two m64n64 fp32 accumulator pairs (x_h w | x_l w_h for both 64-channel halves of N) = 128 per thread, inside
// the 168 that __launch_bounds__(384, 1) leaves (0 spill bytes: tests/test_wide_tower_plan_cpu.py reads the SASS).
//
// Pipeline: per layer 18 weight stages (9 taps x 2 K-halves, 32 KB each) stream from L2 through the two-stage ring by bulk
// copies; thread 0 refills a stage once every warp has released it.  Per stage a warpgroup issues 4 K-steps x 2 N-halves x
// 3 = 24 m64n64k16 MMAs and waits for the previous stage's group.  The M-tiles of a board read each other's rows through
// the halo, so the whole CTA waits for every MMA of layer l before any epilogue of layer l rewrites the planes in place.
// Weight traffic: 576 KB from L2 per board per layer.
//
// CTA pairs (conv_tower_wide_pair_kernel, MZ_TC_WIDE=2 on boards the one-CTA plan refuses, e.g. Gomoku's 15 x 15 and
// 16 x 16): one board per cluster of two CTAs.  CTA rank r owns board rows [r h, min(H, (r + 1) h)), h = ceil(H / 2), and
// keeps the one-CTA layout above for those rows plus one halo board row above and below (local row -1 and `rows`; the
// zero padding row at the board edge), its own fp32 residual rows, its own weight ring and ceil(h S / 64) M-tiles.  The
// numerics, the epilogue and the action-plane table (indexed by the global (y, x)) are the one-CTA kernel's: both are one
// template, so an output element sees the same operands in the same K order.  The epilogue thread that holds a CTA's
// boundary row (CTA 0's last, CTA 1's first) also stores its x_h / x_l into the peer's halo row through distributed shared
// memory, at the peer's plane row (and so the peer's 128B-swizzle phase).  Ordering, per layer l:
//   1. wgmma.wait_group 0, then a cluster barrier (arrive.release / wait.acquire): every MMA of layer l in BOTH CTAs has
//      read its planes, halo rows included, before either epilogue rewrites a row the other CTA's MMAs read;
//   2. the epilogue writes the own rows (generic proxy) and the peer's halo row (generic proxy, st.shared::cluster);
//   3. fence.proxy.async.shared::cluster by every writer, then a cluster barrier: the generic writes of both CTAs, local
//      and remote, are ordered before any wgmma (async proxy) of layer l + 1 reads them.
// The barrier of step 3 after the last layer keeps each CTA resident until its peer has stopped writing into it.  Each CTA
// bumps sat_count for the activations it reads (its rows and halo rows) or stores.  The weight traffic per board doubles
// (each CTA streams its own ring).  Registers: 168, no spills (tests/test_wide_pair_plan_cpu.py reads the SASS).
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

constexpr int kC = kWideC;
constexpr int kRowBytes = 128;                        // one 64-channel K-half of a position, fp16
constexpr int kStageBytes = 256 * kRowBytes;          // 32768: [w_h cout 0..127 | w_l cout 0..127][64 cin]
constexpr int kStagesPerLayer = 18;                   // 9 taps x 2 K-halves
constexpr int kRingStages = 2;
constexpr int kResStride = kC + 8;
constexpr int kMaxMTiles = 3;
constexpr int kMaxThreads = 128 * kMaxMTiles;
constexpr int kRegCap = 168;                          // 65536 / 384 rounded down to the allocation granule
constexpr int kSmemLimit = 232448;
constexpr float kLoScale = 2048.0f, kLoUnscale = 1.0f / 2048.0f;

// The board rows [y0, y0 + rows) a CTA owns: all of them on one CTA; on a pair CTA 0 takes ceil(H / 2), CTA 1 the rest.
// The pair reads its rank with a volatile instruction: the epilogue asks again instead of keeping the geometry live through
// the MMA loop, whose accumulators fill the register budget.
struct WideHalf { int rank, h0, y0, rows; };
template <bool kPair>
MZ_DEVINL WideHalf wide_half(const WideTowerArgs& a) {
    if constexpr (kPair) {
        const int r = (int)cluster_rank(), h0 = (a.H + 1) >> 1;
        return WideHalf{r, h0, r * h0, r ? a.H - h0 : h0};
    } else {
        return WideHalf{0, a.H, 0, a.H};
    }
}

}  // namespace

// One wide tower of one board (kPair = false, one CTA) or of one half of a board (kPair = true, CTA rank r of a cluster of
// two: board rows [y0, y0 + rows), halo rows exchanged through distributed shared memory).  Everything kPair adds folds
// away in the one-CTA instantiation (y0 = 0, rows = H).
template <bool kPair>
MZ_DEVINL void wide_tower_body(const WideTowerArgs& a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const int S = a.S, W = a.W, HW = a.H * a.W;
    const uint32_t plane = (uint32_t)a.plane_bytes;
    const uint32_t s_base = smem_u32(smem);
    const uint32_t s_ring = s_base + 4 * plane;
    float* res = reinterpret_cast<float*>(smem + a.res_off);
    const uint32_t bars = s_base + (uint32_t)a.bar_off;
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (kRingStages + s); };
    const int L = a.n_layers, total = L * kStagesPerLayer;
    const int g = a.g0 + (int)(kPair ? blockIdx.x >> 1 : blockIdx.x);

    if (threadIdx.x == 0) {
        for (int s = 0; s < kRingStages; ++s) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), blockDim.x >> 5); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (uint32_t i = threadIdx.x; i < 4 * plane / 16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    auto load_stage = [&](int q) {                     // thread 0: stage q of the tower into ring slot q % 2
        const int s = q & 1;
        mbar_expect_tx(bar_full(s), kStageBytes);
        bulk_g2s(s_ring + s * kStageBytes,
                 reinterpret_cast<const unsigned char*>(a.layer[q / kStagesPerLayer].w) + (size_t)(q % kStagesPerLayer) * kStageBytes,
                 kStageBytes, bar_full(s));
    };
    if (threadIdx.x == 0) {
        pdl_launch_dependents();
        load_stage(0);                                 // weights are constants; the boards come from the previous kernel
        load_stage(1);
    }
    pdl_wait();

    // ---- the board: NCHW fp32 -> x_h / x_l planes; the first block's residual in fp32.  A CTA of a pair reads its rows
    // and the board rows on either side of them (its halo rows for layer 0).
    const size_t slot = a.gather_parent ? (size_t)g * a.pool_stride + a.gather_parent[g] : (size_t)g;
    const float* src = a.in + slot * (size_t)kC * HW;
    const bool res_in = !a.stem;
    const WideHalf in_half = wide_half<kPair>(a);
    const int y0 = in_half.y0, rows = in_half.rows;
    const int ylo = kPair ? max(y0 - 1, 0) : 0;        // board rows [ylo, ylo + n_read) are read
    const int n_read = kPair ? min(y0 + rows + 1, a.H) - ylo : a.H;
    const int HWr = n_read * W;
    float peak = 0.0f;                                 // largest |activation| this thread read or stored
    for (int i = threadIdx.x; i < kC * HWr; i += blockDim.x) {
        const int c = i / HWr, p = i - c * HWr, yr = p / W, x = p - yr * W;
        const float v = __ldg(src + (kPair ? (size_t)c * HW + (ylo + yr) * W + x : (size_t)i));
        peak = fmaxf(peak, fabsf(v));
        const int y = ylo + yr - y0;                   // my row (-1 and `rows`: halo rows)
        const int row = 1 + (y + 1) * S + x;
        const uint32_t off = (uint32_t)(row * kRowBytes + ((((c & 63) >> 3) ^ (row & 7)) << 4) + (c & 7) * 2);
        split_store(smem + (c >> 6) * plane + off, smem + (2 + (c >> 6)) * plane + off, v);
        if (res_in && (!kPair || (y >= 0 && y < rows))) res[(y * S + x) * kResStride + c] = v;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic smem writes -> wgmma readers
    __syncthreads();

    const int r0 = 16 * (warp & 3) + (lane >> 2);      // accumulator rows r0, r0 + 8 of my M-tile; channels 8 j + cq (+1)
    const int cq = 2 * (lane & 3);
    const int i0 = 64 * wg + r0;                       // interior row of accumulator row r0
    float act_scale = 0.0f;
    if (a.layer[0].action_table) act_scale = __fdiv_rn((float)a.action[g], (float)a.A);
    const uint32_t plane16 = plane >> 4;
    const uint32_t a16 = ((s_base + (uint32_t)((1 + S + 64 * wg) * kRowBytes)) >> 4) | kDescLoFlags;   // my M-tile, plane 0
    const uint32_t ring16 = (s_ring >> 4) | kDescLoFlags;
    float dm[2][32], dl[2][32];                        // x_h (w_h + w_l) | x_l w_h, for the two 64-channel halves of N
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
            const int tap = t >> 1, kh = t & 1;
            mbar_wait(bar_full(q & 1), (uint32_t)((q >> 1) & 1));
            const int shift = (tap / 3 - 1) * S + (tap % 3 - 1);
            const uint32_t ah = a16 + (uint32_t)kh * plane16 + (uint32_t)(shift * (kRowBytes / 16));
            const uint32_t al = ah + 2 * plane16;
            const uint32_t b16 = ring16 + (uint32_t)((q & 1) * (kStageBytes / 16));
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
                for (int nh = 0; nh < 2; ++nh) {
                    const uint32_t bh = b16 + (uint32_t)(nh * (64 * kRowBytes / 16) + ks * 2);     // w_h rows; w_l 128 further
                    const uint32_t first = (t | ks) != 0;
                    wgmma_m64n64k16(dm[nh], ah + ks * 2, bh, first);
                    wgmma_m64n64k16(dm[nh], ah + ks * 2, bh + (uint32_t)(128 * kRowBytes / 16), 1);
                    wgmma_m64n64k16(dl[nh], al + ks * 2, bh, first);
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
        if constexpr (kPair) cluster_barrier();        // every M-tile's MMAs of layer l in both CTAs are complete
        else __syncthreads();                          // every M-tile's MMAs of layer l are complete: rows may be rewritten

        const int bl = l - a.stem;                     // conv index inside the blocks (-1: the stem)
        const bool add_res = bl >= 0 && (bl & 1);
        const bool keep = l + 1 < L && (bl < 0 || (bl & 1));       // this output is the input of a block
        const bool last = l == L - 1;
        const WideHalf me = wide_half<kPair>(a);
        const int y0 = me.y0, interior = me.rows * S;
        // pair: my boundary row (CTA 0's last, CTA 1's first) also goes to the peer's halo row, `peer_shift` plane rows away
        const uint32_t peer_base = kPair ? map_to_cta(s_base, (uint32_t)(me.rank ^ 1)) : 0u;
        const int peer_shift = (me.rank ? me.h0 : -me.h0) * S;              // (y0 - the peer's y0) S
        const int halo_y = me.rank ? 0 : me.rows - 1;
        const float* table = ly.action_table;
        float* dst = a.out + (size_t)g * kC * HW;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = i0 + 8 * h;
            if (i >= interior) continue;               // masked rows
            const int y = i / S, x = i - y * S;
            const bool live = x < W;
            const int row = 1 + S + i;
#pragma unroll
            for (int nh = 0; nh < 2; ++nh)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 64 * nh + 8 * j + cq;
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int k = 4 * j + 2 * h + e;
                        float u = fmaf(dl[nh][k], kLoUnscale, dm[nh][k]) * __ldg(ly.scale + c + e) + (ly.bias ? __ldg(ly.bias + c + e) : 0.0f);
                        if (add_res) u += res[i * kResStride + c + e];
                        if (table && live) u = fmaf(act_scale, __ldg(table + (size_t)((y0 + y) * W + x) * kC + c + e), u);
                        u = fmaxf(u, 0.0f);
                        if (!live) u = 0.0f;           // the zero column stays zero
                        peak = fmaxf(peak, fabsf(u));
                        v[e] = u;
                    }
                    if (keep) *reinterpret_cast<float2*>(res + i * kResStride + c) = make_float2(v[0], v[1]);
                    if (last) {
                        if (live) {
                            dst[(size_t)c * HW + (y0 + y) * W + x] = v[0];
                            dst[(size_t)(c + 1) * HW + (y0 + y) * W + x] = v[1];
                        }
                    } else {
                        const uint32_t off = (uint32_t)(row * kRowBytes + ((j ^ (row & 7)) << 4) + 2 * cq);
                        const uint32_t hw = pack_f16x2(v[0], v[1]);
                        const float2 hf = unpack_f16x2(hw);
                        const uint32_t lw = pack_f16x2((v[0] - hf.x) * kLoScale, (v[1] - hf.y) * kLoScale);
                        *reinterpret_cast<uint32_t*>(smem + nh * plane + off) = hw;
                        *reinterpret_cast<uint32_t*>(smem + (2 + nh) * plane + off) = lw;
                        if constexpr (kPair) {
                            if (y == halo_y) {                 // the peer's plane row, with its own swizzle phase
                                const int prow = row + peer_shift;
                                const uint32_t poff = (uint32_t)(prow * kRowBytes + ((j ^ (prow & 7)) << 4) + 2 * cq);
                                st_cluster_u32(peer_base + nh * plane + poff, hw);
                                st_cluster_u32(peer_base + (2 + nh) * plane + poff, lw);
                            }
                        }
                    }
                }
        }
        if constexpr (kPair) {                         // my local and remote generic writes -> both CTAs' wgmma readers
            asm volatile("fence.proxy.async.shared::cluster;" ::: "memory");
            cluster_barrier();                         // after the last layer: the peer no longer writes into my planes
        } else {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
        }
    }
    if (peak > 65504.0f && a.sat_count) atomicAdd(a.sat_count, 1);
}

__global__ void __launch_bounds__(kMaxThreads, 1) conv_tower_wide_kernel(const __grid_constant__ WideTowerArgs a) {
    wide_tower_body<false>(a);
}

// launched in clusters of two CTAs (launch_chained_cluster), grid 2n: cluster k runs board g0 + k
__global__ void __launch_bounds__(kMaxThreads, 1) conv_tower_wide_pair_kernel(const __grid_constant__ WideTowerArgs a) {
    wide_tower_body<true>(a);
}

namespace {

enum WideBudgetFit { kFits, kTooManyMTiles, kOverSmem, kOverRing };

// Budget of one CTA holding `board_rows` board rows of width W (plus a zero / halo row above and below): the one-CTA
// kernel's whole board, or one half of a pair's
WideBudgetFit wide_budget(int board_rows, int W, int sm_count, int layers, WideTowerPlan* p) {
    const int S = W + 1, interior = board_rows * S;
    const int m_tiles = (interior + 63) / 64;
    if (m_tiles > kMaxMTiles) return kTooManyMTiles;
    const int rows = ((board_rows + 2) * S + 1 + 7) & ~7;
    const size_t planes = (size_t)4 * rows * kRowBytes;
    const size_t res = (size_t)interior * kResStride * 4;
    const size_t smem = planes + (size_t)kRingStages * kStageBytes + res + 8 * 2 * kRingStages;
    if (smem > (size_t)kSmemLimit) return kOverSmem;
    // masked output rows read at most 2 S + 64 m_tiles + 1 rows from the last plane's start: they must stay inside the ring
    if ((2 * S + 64 * m_tiles + 1 - rows) * kRowBytes > kRingStages * kStageBytes) return kOverRing;
    p->m_tiles = m_tiles;
    p->threads = 128 * m_tiles;
    p->rows = rows;
    p->stages = kRingStages;
    p->smem = smem;
    p->layers = layers;
    const int by_smem = (int)(233472 / (smem + 2048));           // 228 KB per SM; per CTA 1 KB reserved + 1 KB static (alignment)
    const int by_regs = 65536 / (p->threads * kRegCap);
    p->ctas_per_sm = std::min(std::min(by_smem, by_regs), 2048 / p->threads);
    p->wave = p->ctas_per_sm * sm_count;
    p->launches = 1;                                   // one CTA (or CTA pair) per board: any batch is one launch
    p->reg_cap = kRegCap;
    return kFits;
}

// the launcher's checks of the arguments and the layout fields of one CTA holding `board_rows` board rows
bool wide_args_fill(WideTowerArgs& a, const WideTowerPlan& p, int board_rows) {
    if (a.n_layers != p.layers || a.n < 1) return false;
    for (int l = 1; l < a.n_layers; ++l) if (a.layer[l].action_table) return false;   // a table belongs to the stem
    if (a.layer[0].action_table && (!a.stem || !a.action)) return false;
    a.S = a.W + 1;
    a.plane_bytes = p.rows * kRowBytes;
    a.res_off = 4 * a.plane_bytes + kRingStages * kStageBytes;
    a.bar_off = a.res_off + board_rows * a.S * kResStride * 4;
    return true;
}

}  // namespace

bool wide_tower_plan(int n, int C, int H, int W, int layers, int sm_count, WideTowerPlan* p, const char** why) {
    *p = WideTowerPlan{};
    if (C != kC) { *why = "the wide towers take 128 channels"; return false; }
    if (n < 1 || H < 1 || W < 1 || sm_count < 1) { *why = "empty shape"; return false; }
    if (layers < 1 || layers > kWideMaxLayers) { *why = "1 to 21 layers (a stem and up to 10 blocks)"; return false; }
    switch (wide_budget(H, W, sm_count, layers, p)) {
        case kTooManyMTiles: *why = "board too large: H x (W + 1) exceeds the 192 rows of three M-tiles"; return false;
        case kOverSmem: *why = "board too large: activations, weight ring and residual exceed shared memory"; return false;
        case kOverRing: *why = "tap windows overrun the ring"; return false;
        case kFits: break;
    }
    return true;
}

bool wide_pair_plan(int n, int C, int H, int W, int layers, int sm_count, WideTowerPlan* p, const char** why) {
    *p = WideTowerPlan{};
    if (C != kC) { *why = "the wide towers take 128 channels"; return false; }
    if (n < 1 || H < 1 || W < 1 || sm_count < 1) { *why = "empty shape"; return false; }
    if (H < 2) { *why = "a CTA pair splits the board rows: H >= 2"; return false; }
    if (layers < 1 || layers > kWideMaxLayers) { *why = "1 to 21 layers (a stem and up to 10 blocks)"; return false; }
    const int h = (H + 1) / 2;
    switch (wide_budget(h, W, sm_count, layers, p)) {
        case kTooManyMTiles:
            *why = "board too large: ceil(H / 2) x (W + 1) exceeds the 192 rows of three M-tiles per CTA"; return false;
        case kOverSmem:
            *why = "board too large: a half's activations, weight ring and residual exceed shared memory"; return false;
        case kOverRing: *why = "tap windows overrun the ring"; return false;
        case kFits: break;
    }
    p->pair_rows0 = h;
    p->wave = p->ctas_per_sm * sm_count / 2;           // boards (CTA pairs) per wave, as planned: the GPCs may hold fewer
    return true;
}

cudaError_t launch_wide_tower(WideTowerArgs a, const WideTowerPlan& p, cudaStream_t stream) {
    static size_t attr_smem = 0;
    if (attr_smem < p.smem) {
        cudaError_t e = cudaFuncSetAttribute(conv_tower_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
        if (e != cudaSuccess) return e;
        attr_smem = p.smem;
    }
    if (p.pair_rows0 || !wide_args_fill(a, p, a.H)) return cudaErrorInvalidValue;
    cudaError_t e = launch_chained(conv_tower_wide_kernel, dim3(a.n), dim3(p.threads), p.smem, stream, a);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

cudaError_t launch_wide_pair_tower(WideTowerArgs a, const WideTowerPlan& p, cudaStream_t stream) {
    static size_t attr_smem = 0;
    if (attr_smem < p.smem) {
        cudaError_t e = cudaFuncSetAttribute(conv_tower_wide_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
        if (e != cudaSuccess) return e;
        attr_smem = p.smem;
    }
    if (p.pair_rows0 != (a.H + 1) / 2 || !wide_args_fill(a, p, p.pair_rows0)) return cudaErrorInvalidValue;
    cudaError_t e = launch_chained_cluster(conv_tower_wide_pair_kernel, dim3(2 * a.n), dim3(p.threads), dim3(2, 1, 1), p.smem,
                                           stream, a);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

}  // namespace mz
