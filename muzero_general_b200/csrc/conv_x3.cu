// Residual towers on the tensor cores at fp32-grade accuracy ("x3" mode, the default for 64-channel board nets).
//
// The reference evaluates its networks in fp32 (models.py:206-231).  An f16 wgmma only takes 16-bit operands, so
// every fp32 operand is split in two 16-bit terms and three of the four partial products are kept:
//
//     x = x_h + x_l/2^11   x_h = fp16(x) (11 significant bits),  x_l = fp16((x - x_h) 2^11) (11 more bits; the scale keeps
//                          the remainder a NORMAL fp16 number wherever x_h is one, so small activations keep 22 bits too)
//     w = (w_h + w_l)/s    s = a power of two per output channel that brings the row's largest |w| into [1, 2);
//                          w_h = fp16(w s), w_l = fp16(w s - w_h): 22 significant bits relative to the row maximum
//     conv = sum x_h w_h + x_h w_l + x_l w_h                    (the dropped x_l w_l term is 2^-22 of |x||w|)
//
// Products of 16-bit operands are exact in fp32 and the accumulation is fp32, so the result carries ~2^-20 relative
// error per term: the class of an fp32 FMA loop in a different summation order, and two to three orders of magnitude
// inside the 2e-4 network tolerance of the test-suite.  (An f16 MMA takes fp16 or bf16 operands but not one of each,
// hence the scaled fp16 remainder.)  Activations beyond the fp16 range (|x| > 65504) saturate x_h (and possibly x_l):
// they leave the accuracy contract, so the epilogue tracks the largest |x| it stores and bumps a counter the host
// checks after every search (ResNetDevice falls back to the fp32 CUDA-core towers, resnet.cu).
//
// Cost: 3 MMAs per 16-channel K-step instead of 1.  x_h w_h and x_h w_l accumulate into the same registers (both are
// on the scale of w); x_l w_h goes to a second accumulator, and the epilogue forms acc + acc_l / 2^11.
//
// Kernel structure (one CTA per SM, up to two tiles = four boards per CTA, all layers of a tower in one launch):
//   weights   [9 taps][128 rows: w_h couts | w_l couts][64 cin fp16], 128B-swizzled, 144 KB, ONE slot set refilled
//             tap by tap for layer l+1 while the last tile of layer l still multiplies
//   X         the CTA's boards as two swizzled fp16 planes (x_h, x_l), 2 x 36 KB, updated IN PLACE: a layer's
//             output may overwrite its input because (a) the warpgroup that owns a board rewrites it only after its own
//             MMAs on the board have completed, (b) other boards' MMAs only read this board's rows for their padding
//             outputs, which are stored as zeros, and (c) the residual stream lives in the epilogue threads' REGISTERS
//             in fp32 (each thread owns two board positions x 16 channels through the whole tower), so a block input
//             never has to stay in memory
//   D         registers: 2 x 32 fp32 per thread (m64n64 accumulators of the board's warpgroup)
// Warp roles: warpgroup 2k + b (warps 4(2k+b)..+3) multiplies and finishes board b of tile k and bulk-stores it after
// the last layer.  Warp 0 also issues the bulk loads: the inputs and layer 0's weights up front, and layer l+1's weights
// after its own epilogue of layer l, once every warpgroup has finished its MMAs of layer l (which it has to wait for
// anyway before it can multiply layer l+1).  A separate producer warp would cap the 128 MMA threads below 128 registers.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>

#include "conv_tc.h"
#include "launch.h"
#include "pipeline.h"
#include "tc_common.cuh"

namespace mz {

namespace {

using namespace tc;

constexpr int kC = 64;
constexpr int kPos = 64;
constexpr int kBoards = 2;                                   // boards per tile
constexpr int kHalo = 16;
constexpr int kRowBytes = 128;
constexpr int kTiles = 2;                                    // tiles per CTA
constexpr int kRowsX = kTiles * kBoards * kPos + 2 * kHalo;  // 288
constexpr int kPlaneBytes = kRowsX * kRowBytes;              // 36864
constexpr int kTapBytes = 128 * kRowBytes;                   // 16384
constexpr int kWBytes = 9 * kTapBytes;                       // 147456
constexpr int kBoardPlane = kPos * kRowBytes;                // 8192: one plane of one board
constexpr int kBoardBytes = 2 * kBoardPlane;                 // 16384: x_h plane | x_l plane
constexpr float kLoScale = 2048.0f, kLoUnscale = 1.0f / 2048.0f;
constexpr int kConsumerWarps = 4 * kTiles * kBoards;         // one warpgroup per board
constexpr int kThreads = 32 * kConsumerWarps;

struct SmemX {
    static constexpr int w = 0;
    static constexpr int hi = kWBytes;
    static constexpr int lo = hi + kPlaneBytes;
    static constexpr int bias = lo + kPlaneBytes;                          // [kTowerMaxLayers][64]
    static constexpr int scale = bias + kTowerMaxLayers * kC * 4;          // [kTowerMaxLayers][64]
    static constexpr int bars = scale + kTowerMaxLayers * kC * 4;
    static constexpr int total = bars + 32 * 8;
};
static_assert(SmemX::total <= 232448, "shared memory budget");
static_assert(SmemX::hi % 1024 == 0 && SmemX::lo % 1024 == 0, "activation planes must keep the 1024-byte swizzle phase");

// x = x_h + x_l / 2^11 from the two packed planes
MZ_DEVINL float2 join_split(uint32_t h, uint32_t l) {
    const float2 hf = unpack_f16x2(h), lf = unpack_f16x2(l);
    return make_float2(fmaf(lf.x, kLoUnscale, hf.x), fmaf(lf.y, kLoUnscale, hf.y));
}

// boards hold two 8 KB planes (x_h | x_l); the host side types the buffers float*: 4096 float slots per board
MZ_DEVINL const unsigned char* x3_board(const TowerArgs& a, int buf, int g) {
    const unsigned char* base = reinterpret_cast<const unsigned char*>(a.buf[buf]);
    if (buf == 0 && a.gather_parent)
        return base + ((size_t)g * a.pool_stride + a.gather_parent[g]) * (size_t)kBoardBytes;
    return base + (size_t)g * kBoardBytes;
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 1) conv_tower_x3_kernel(const __grid_constant__ TowerArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int kStampBase = kTowerMaxLayers * kTiles * 4;     // timeline: [+0] kernel entry, [+1] setup done, [+2] outputs stored
    if (a.timeline && blockIdx.x == 0 && threadIdx.x == 0) a.timeline[kStampBase] = clock64();
    const uint32_t s_base = smem_u32(smem);
    const uint32_t s_w = s_base + SmemX::w, s_hi = s_base + SmemX::hi, s_lo = s_base + SmemX::lo;
    float* s_bias = reinterpret_cast<float*>(smem + SmemX::bias);
    float* s_scale = reinterpret_cast<float*>(smem + SmemX::scale);
    const uint32_t bars = s_base + SmemX::bars;
    auto bar_w_full = [&](int tap) { return bars + 8u * tap; };
    auto bar_w_empty = [&](int tap) { return bars + 8u * (9 + tap); };
    auto bar_in_full = [&](int k) { return bars + 8u * (18 + k); };         // input boards of my k-th tile landed

    const int n_tiles = (a.n + kBoards - 1) / kBoards;
    const int tile0 = (int)blockIdx.x * kTiles;
    const int my_tiles = min(kTiles, n_tiles - tile0);
    const int L = a.n_layers;

    // ---- one-time setup: zero halos of both planes, biases / scales, barriers
    for (int i = threadIdx.x; i < 2 * 2 * kHalo * (kRowBytes / 16); i += kThreads) {
        const int chunk = i % (kRowBytes / 16), r = (i / (kRowBytes / 16)) % (2 * kHalo), pl = i / ((kRowBytes / 16) * 2 * kHalo);
        const int row = r < kHalo ? r : kRowsX - 2 * kHalo + r;
        reinterpret_cast<uint4*>(smem + SmemX::hi + pl * kPlaneBytes + row * kRowBytes)[chunk] = make_uint4(0, 0, 0, 0);
    }
    if (my_tiles < kTiles) {
        // a CTA with one tile: the rows of the missing tile are read by the last tap windows of tile 0
        for (int i = threadIdx.x; i < 2 * kBoards * kPos * (kRowBytes / 16); i += kThreads) {
            const int chunk = i % (kRowBytes / 16), r = (i / (kRowBytes / 16)) % (kBoards * kPos), pl = i / ((kRowBytes / 16) * kBoards * kPos);
            reinterpret_cast<uint4*>(smem + SmemX::hi + pl * kPlaneBytes + (kHalo + kBoards * kPos + r) * kRowBytes)[chunk] = make_uint4(0, 0, 0, 0);
        }
    }
    for (int i = threadIdx.x; i < L * kC; i += kThreads) {
        const float* b = a.layer[i / kC].bias;
        const float* sc = a.layer[i / kC].scale;
        s_bias[i] = b ? b[i % kC] : 0.0f;
        s_scale[i] = sc ? sc[i % kC] : 1.0f;
    }
    if (threadIdx.x == 0) {
        // every warp of the warpgroups with a tile arrives once per layer
        for (int t = 0; t < 9; ++t) { mbar_init(bar_w_full(t), 1); mbar_init(bar_w_empty(t), 4 * kBoards * my_tiles); }
        for (int k = 0; k < kTiles; ++k) mbar_init(bar_in_full(k), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (a.timeline && blockIdx.x == 0 && threadIdx.x == 0) a.timeline[kStampBase + 1] = clock64();

    auto load_weights = [&](int l) {                  // warp 0, lane = tap
        mbar_expect_tx(bar_w_full(lane), kTapBytes);
        bulk_g2s(s_w + lane * kTapBytes, reinterpret_cast<const unsigned char*>(a.layer[l].w) + (size_t)lane * kTapBytes, kTapBytes,
                 bar_w_full(lane));
    };
    if (warp == 0) {
        pdl_launch_dependents();
        if (lane < 9) load_weights(0);
        pdl_wait();                                    // weights are constants; the boards come from the previous kernel
        const int in_buf = a.layer[0].in_buf;
        for (int k = 0; k < my_tiles; ++k) {
            const int b0 = (tile0 + k) * kBoards;
            const int nb = min(kBoards, a.n - b0);
            if (lane == 0) mbar_expect_tx(bar_in_full(k), (uint32_t)nb * kBoardBytes);
            __syncwarp();
            if (lane < 2 * nb) {                       // lane = board * 2 + plane
                const int b = lane >> 1, pl = lane & 1;
                bulk_g2s((pl ? s_lo : s_hi) + (kHalo + (k * kBoards + b) * kPos) * kRowBytes,
                         x3_board(a, in_buf, a.g0 + b0 + b) + pl * kBoardPlane, kBoardPlane, bar_in_full(k));
            }
        }
        __syncwarp();
    }
    // ================= MMA + epilogue: warpgroup wg owns board wg & 1 of tile wg >> 1, for the whole tower =================
    const int wg = warp >> 2;
    const int k = wg >> 1, b = wg & 1;
    if (k >= my_tiles) return;
    pdl_wait();                                        // reads a.action (written by the tree kernel)
    const int r0 = 16 * (warp & 3) + (lane >> 2);      // accumulator rows (board positions) r0, r0 + 8; channels 8 j + cq (+1)
    const int cq = 2 * (lane & 3);
    const int sw = lane >> 2;                          // chunk c of the row is stored at chunk c ^ sw
    const int gl = (tile0 + k) * kBoards + b;          // board inside this launch
    const int g = a.g0 + gl;
    const bool stamp = a.timeline && blockIdx.x == 0 && b == 0 && (threadIdx.x & 127) == 0;
    const int brow = kHalo + (k * kBoards + b) * kPos;
    bool live[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int p = r0 + 8 * h, y = p / 8 - 1, x = p % 8;
        live[h] = (y >= 0 && y < a.H && x < a.W) && gl < a.n;
    }
    // this thread's 4-byte slot (row r0 + 8 h, channels 8 j + cq, +1) in a plane; i = 4 j + 2 h + e indexes the accumulators
    auto slot_off = [&](int h, int j) { return (brow + r0 + 8 * h) * kRowBytes + ((j ^ sw) << 4) + 2 * cq; };
    float res[32];                                     // residual stream of this thread's positions / channels, fp32
#pragma unroll
    for (int i = 0; i < 32; ++i) res[i] = 0.0f;
    float peak = 0.0f;                                 // largest |activation| this thread read or stored
    const bool res_from_input = L >= 2 && a.layer[1].res_buf >= 0;      // the tower starts with a block
    const bool res_external = a.layer[0].res_buf >= 0;                  // single conv with a residual (debug entry)
    mbar_wait(bar_in_full(k), 0);
    if (res_from_input && gl < a.n) {                  // a missing board's rows were never loaded
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float2 xf = join_split(*reinterpret_cast<const uint32_t*>(smem + SmemX::hi + slot_off(h, j)),
                                             *reinterpret_cast<const uint32_t*>(smem + SmemX::lo + slot_off(h, j)));
                res[4 * j + 2 * h] = xf.x;
                res[4 * j + 2 * h + 1] = xf.y;
                peak = fmaxf(peak, fmaxf(fabsf(xf.x), fabsf(xf.y)));
            }
    } else if (res_external && gl < a.n) {
        const unsigned char* rb = x3_board(a, a.layer[0].res_buf, g);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int off = (r0 + 8 * h) * kRowBytes + ((j ^ sw) << 4) + 2 * cq;
                const float2 xf = join_split(__ldg(reinterpret_cast<const unsigned int*>(rb + off)),
                                             __ldg(reinterpret_cast<const unsigned int*>(rb + kBoardPlane + off)));
                res[4 * j + 2 * h] = xf.x;
                res[4 * j + 2 * h + 1] = xf.y;
                peak = fmaxf(peak, fmaxf(fabsf(xf.x), fabsf(xf.y)));
            }
    }
    const uint32_t ah16 = ((s_hi + (uint32_t)(brow * kRowBytes)) >> 4) | kDescLoFlags;
    const uint32_t al16 = ((s_lo + (uint32_t)(brow * kRowBytes)) >> 4) | kDescLoFlags;
    const uint32_t w16 = (s_w >> 4) | kDescLoFlags;
    for (int l = 0; l < L; ++l) {
        const TowerLayer& ly = a.layer[l];
        const float* bias = s_bias + l * kC;
        const float* scale = s_scale + l * kC;
        const bool last = l == L - 1;
        const bool add_res = ly.res_buf >= 0;
        const bool keep = l + 2 < L && a.layer[l + 2].res_buf >= 0;     // this output is the input of a block
        float act_scale = 0.0f;
        if (gl < a.n && ly.action_table) act_scale = __fdiv_rn((float)a.action[g], (float)a.A);
        // the action table entries of this thread (dynamics stem) go to the idle residual registers before the MMAs, so
        // the loads overlap them.  The table sits on the stem, before the first block: the registers are free (the
        // launcher rejects a table anywhere else)
        const bool table = ly.action_table != nullptr;
        if (table) {
#pragma unroll
            for (int i = 0; i < 32; ++i)
                res[i] = __ldg(ly.action_table + (size_t)(r0 + 8 * ((i >> 1) & 1)) * kC + 8 * (i >> 2) + cq + (i & 1));
        }
        if (stamp) a.timeline[(l * kTiles + k) * 4 + 0] = clock64();
        float dm[32], dl[32];                          // x_h (w_h + w_l) | x_l w_h
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            mbar_wait(bar_w_full(tap), (uint32_t)(l & 1));
            constexpr int kRow16 = kRowBytes / 16;
            const int shift = (tap / 3 - 1) * 8 + (tap % 3 - 1);
#pragma unroll
            for (int ks = 0; ks < kC / 16; ++ks) {
                const uint32_t off = (uint32_t)(shift * kRow16 + ks * 2);
                const uint32_t bh = w16 + (uint32_t)(tap * (kTapBytes / 16) + ks * 2);     // w_h rows; w_l rows 64 further
                wgmma_m64n64k16(dm, ah16 + off, bh, (tap | ks) != 0);
                wgmma_m64n64k16(dm, ah16 + off, bh + (uint32_t)(kC * kRowBytes / 16), 1);
                wgmma_m64n64k16(dl, al16 + off, bh, (tap | ks) != 0);
            }
        }
        wgmma_commit();
        if (stamp) a.timeline[(l * kTiles + k) * 4 + 1] = clock64();
        wgmma_wait_all();
        if (stamp) a.timeline[(l * kTiles + k) * 4 + 2] = clock64();
        __syncwarp();
        if (lane == 0)
            for (int tap = 0; tap < 9; ++tap) mbar_arrive(bar_w_empty(tap));
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int c = 8 * (i >> 2) + cq + (i & 1);
            float v = fmaf(dl[i], kLoUnscale, dm[i]) * scale[c] + bias[c];
            if (add_res) v += res[i];
            if (table) v = fmaf(act_scale, res[i], v);
            if (ly.relu) v = fmaxf(v, 0.0f);
            if (!live[(i >> 1) & 1]) v = 0.0f;        // padding rows and missing boards stay zero
            if (keep) res[i] = v;
            peak = fmaxf(peak, fabsf(v));
            dm[i] = v;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float v0 = dm[4 * j + 2 * h], v1 = dm[4 * j + 2 * h + 1];
                const uint32_t hw = pack_f16x2(v0, v1);
                const float2 hf = unpack_f16x2(hw);
                *reinterpret_cast<uint32_t*>(smem + SmemX::hi + slot_off(h, j)) = hw;
                *reinterpret_cast<uint32_t*>(smem + SmemX::lo + slot_off(h, j)) = pack_f16x2((v0 - hf.x) * kLoScale, (v1 - hf.y) * kLoScale);
            }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic smem writes -> wgmma / bulk-copy readers
        warpgroup_sync(wg);
        if (stamp) a.timeline[(l * kTiles + k) * 4 + 3] = clock64();
        if (warp == 0 && l + 1 < L) {
            if (lane < 9) {
                mbar_wait(bar_w_empty(lane), (uint32_t)(l & 1));             // every warpgroup is done with this tap
                load_weights(l + 1);
            }
            __syncwarp();
        }
        if (last && (threadIdx.x & 127) == 0 && gl < a.n) {
            unsigned char* dst = reinterpret_cast<unsigned char*>(a.buf[ly.out_buf]) + (size_t)g * kBoardBytes;
            bulk_s2g(dst, s_hi + (uint32_t)(brow * kRowBytes), kBoardPlane);
            bulk_s2g(dst + kBoardPlane, s_lo + (uint32_t)(brow * kRowBytes), kBoardPlane);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
            if (stamp) a.timeline[kStampBase + 2] = clock64();
        }
    }
    if (peak > 65504.0f && a.sat_count) atomicAdd(a.sat_count, 1);
}

// Any batch: chunks of at most sm_count * 4 boards, one launch each (balanced, multiples of one CTA's four boards).
cudaError_t launch_conv_tower_x3(const TowerArgs& args, int sm_count, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(conv_tower_x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemX::total);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    if (args.n_layers < 1 || args.n_layers > kTowerMaxLayers) return cudaErrorInvalidValue;
    for (int l = 0; l < args.n_layers; ++l) {          // block structure: a residual is the input of the layer before
        const TowerLayer& t = args.layer[l];
        if (l > 0 && t.in_buf != args.layer[l - 1].out_buf) return cudaErrorInvalidValue;
        if (l > 0 && t.res_buf >= 0 && t.res_buf != args.layer[l - 1].in_buf) return cudaErrorInvalidValue;
        // an action table belongs to a stem: first layer, no residual, not the first conv of a block (the kernel parks the
        // table row in the residual registers, which must be idle)
        if (t.action_table && (l > 0 || t.res_buf >= 0 || (args.n_layers >= 2 && args.layer[1].res_buf >= 0))) return cudaErrorInvalidValue;
    }
    // profiling: MZ_X3_TIMELINE=<file> appends CTA 0's per-layer clock64 stamps of every launch (synchronous; never
    // set inside a graph capture - use MZ_NO_GRAPH=1)
    static const char* timeline_path = getenv("MZ_X3_TIMELINE");
    static long long* d_timeline = nullptr;
    constexpr int kTimelineWords = kTowerMaxLayers * kTiles * 4 + 4;
    if (timeline_path && !d_timeline && cudaMalloc(&d_timeline, kTimelineWords * sizeof(long long)) != cudaSuccess)
        return cudaErrorMemoryAllocation;
    const int per_launch = sm_count * kTiles * kBoards;
    const int chunks = (args.n + per_launch - 1) / per_launch;
    int per = (args.n + chunks - 1) / chunks;
    per = (per + kTiles * kBoards - 1) / (kTiles * kBoards) * (kTiles * kBoards);
    for (int g0 = 0; g0 < args.n; g0 += per) {
        TowerArgs a = args;
        a.g0 = args.g0 + g0;
        a.n = (args.n - g0 < per) ? args.n - g0 : per;
        const int n_tiles = (a.n + kBoards - 1) / kBoards;
        const int grid = (n_tiles + kTiles - 1) / kTiles;
        a.timeline = timeline_path ? d_timeline : nullptr;
        cudaError_t e = launch_chained(conv_tower_x3_kernel, dim3(grid), dim3(kThreads), SmemX::total, stream, a);
        if (e != cudaSuccess) return e;
        if (timeline_path) {
            long long h[kTimelineWords];
            if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
            if ((e = cudaMemcpy(h, d_timeline, sizeof(h), cudaMemcpyDeviceToHost)) != cudaSuccess) return e;
            if (FILE* f = fopen(timeline_path, "a")) {
                const long long* st = h + kTowerMaxLayers * kTiles * 4;
                fprintf(f, "launch boards=%d layers=%d entry=%lld setup=%lld stored=%lld\n", a.n, a.n_layers, st[0] - h[0], st[1] - h[0], st[2] - h[0]);
                for (int l = 0; l < a.n_layers; ++l)
                    for (int k = 0; k < kTiles; ++k) {
                        const long long* t = h + (l * kTiles + k) * 4;
                        fprintf(f, "%d %d %lld %lld %lld %lld\n", l, k, t[0] - h[0], t[1] - h[0], t[2] - h[0], t[3] - h[0]);
                    }
                fclose(f);
            }
        }
    }
    return cudaGetLastError();
}

int conv_x3_launches(int n, int sm_count) { return (n + sm_count * kTiles * kBoards - 1) / (sm_count * kTiles * kBoards); }

}  // namespace mz
