// Heads of the residual networks (models.py:530-553 rescale, reward / value / policy heads) as device code shared by
// heads_kernel (resnet.cu) and the fused small-network search kernel (small_search.cu).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "fc_net.cuh"
#include "launch.h"

namespace mz {

// Board layouts of the tensor-core towers (conv_tc.cu / conv_x3.cu): kLayoutF16 = one fp16 plane of 4096 halves,
// kLayoutSplit = two fp16 planes, x_h then x_l with x ~ x_h + x_l / 2^11 (8192 halves = 4096 float slots per board).
enum { kLayoutDense = 0, kLayoutF16 = 1, kLayoutSplit = 2 };
constexpr float kSplitLoScale = 2048.0f, kSplitLoUnscale = 1.0f / 2048.0f;

// ------------------------------------------------------------------------------------------
// Heads: conv1x1(+bias) -> flatten (c,h,w) -> MLP -> logits (-> support_to_scalar), plus the
// per-(sample, channel) min-max rescale of the state (models.py:530-553).  One CTA per sample.
// ------------------------------------------------------------------------------------------
struct HeadDesc {
    int rc;                    // reduced channels
    int w1_off, b1_off;        // conv1x1 weight [rc][C], bias [rc]
    MlpDesc mlp;               // transposed layers in the same blob
    int n_out;                 // logits
};

struct HeadsArgs {
    const float* x;            // [n, C, HW] input state (raw trunk output)
    const float* blob;
    int n, C, HW, S;
    unsigned hw_inv;           // ceil(2^32 / HW) (0 when HW == 1): divisions by HW become a multiply-high
    int g0;                    // samples [g0, g0 + n), arrays addressed by the global index
    int n_heads;
    HeadDesc head[2];
    float* logits[2];          // [n, n_out] or nullptr
    float* scalar[2];          // [n] support_to_scalar or nullptr
    // optional rescale of x into the hidden pool / a plain buffer
    float* rescaled;           // [n, C*HW] or nullptr
    float* pool_hidden;        // pool mode target
    int pool_stride, out_slot;
    int smem_floats;
    int p64c4, W;              // kLayoutF16 / kLayoutSplit: input (and pool target) use the tensor-core board layout
    float* state_p64c4;        // [n, 4096 fp16] rescaled state in P64C8 (input of the prediction tower), or nullptr
    int w_lo, w_floats;        // slice of the head blob this launch needs (staged in shared memory)
    int warp_floats;           // per-warp scratch: x tile + two activation vectors
};

// offset (in fp16 elements) of (channel c, dense position p) inside one P64S state of 4096 halves: position-major
// rows of 64 channels, the 8-channel chunks of a row XOR-ed with (padded position % 8) (conv_tc.cu)
__device__ __forceinline__ int p64c4_index(int c, int p, int W) {
    const int pos = (p / W + 1) * 8 + (p % W);
    return pos * 64 + ((((c >> 3) ^ (pos & 7))) << 3) + (c & 7);
}

// Persistent CTAs (one per SM), 1024 threads = 8 groups of 128: the head weights of this launch are staged
// in shared memory once per CTA, then every GROUP takes one sample at a time (named barriers, groups never
// wait for each other).  x is staged as a [position][channel] tile with 16-byte aligned rows (row stride C+4:
// conflict-free for 128-bit row reads and for per-channel column scans).  Everything that touches global
// memory or the weights moves 16 bytes per instruction: the P64S state is read and written as whole 8-channel
// chunks, conv1x1 reads x rows and weight rows as float4, the FC layers read packed [in/4][out][4] weights and
// float4 activations; index arithmetic with runtime divisors happens once per chunk, not per element.
// The accumulation order of every dot product is ascending input index (as torch's reference loops are
// compared with a tolerance anyway, this only keeps results independent of the vector width).
// GROUP = 128 threads per sample for wide states (Connect4: 64 x 42), GROUP = 32 (one warp per sample, __syncwarp
// instead of named barriers, 4x the samples in flight) when a sample is only a few hundred values (TicTacToe 16 x 9,
// Breakout's 16 x 36 hidden board).
constexpr int kHeadThreads = 1024;

template <int GROUP>
__device__ __forceinline__ void group_bar(int group) {
    if constexpr (GROUP == 32) __syncwarp();
    else asm volatile("bar.sync %0, %1;" ::"r"(group + 1), "r"(GROUP) : "memory");
}

// One sample of a heads launch, executed by one group of GROUP threads (t = thread inside the group): stage x, rescale
// (optional), conv1x1 + MLP + scalarisation of the launch's heads.  `blob` addresses the staged head weights
// (blob[off] = head blob offset off), `scratch` is the group's private shared memory (HeadsArgs::warp_floats floats),
// s_pos the padded-row table of the board layouts (unused for dense states), out_slot the pool slot of the rescaled state.  Shared by heads_kernel and the fused small-network search kernel.
// Resident mode (fused search kernel): `tile` connects the sample to the padded shared-memory board buffers of the towers -
// src: the board's raw state is read from there instead of a.x, dst: the rescaled state is ALSO written there (the
// prediction tower's input), map: dense element c * HW + pos -> offset inside a board buffer, xmap: -> offset inside s_x.
struct HeadsTile { const float* src; float* dst; const int* map; const int* xmap; };

template <int GROUP>
__device__ __forceinline__ void heads_one_sample(const HeadsArgs& a, const float* blob, float* scratch, const unsigned char* s_pos,
                                                 int g, int group, int t, int out_slot, HeadsTile tile = HeadsTile{nullptr, nullptr, nullptr, nullptr}) {
    constexpr int kHeadGroup = GROUP;
    const int C = a.C, HW = a.HW, CP = C + 4;
    float* s_x = scratch;                                            // [HW][C+4]
    float* s_lo = s_x + HW * CP;                                     // [C] channel minimum
    float* s_sc = s_lo + C;                                          // [C] channel scale
    float* s_part = s_sc + C;                                        // [2][2][C] partial extrema
    float* s_act = s_part + 4 * C;                                   // per head: ping | pong
    constexpr int cj = 8;                                            // 8-channel chunks per position (board layout: C = 64)
    // i / HW without a division: __umulhi(i, ceil(2^32 / HW)) is exact for every HW and index a group's tile can hold
    // (tests/test_heads_plan_cpu.py::test_hw_inv_division_is_exact_for_every_index_heads_kernel_takes)
    const unsigned hw_inv = a.hw_inv;                                // filled by the host (0: HW == 1)
    auto div_hw = [&](int i) { return hw_inv ? (int)__umulhi((unsigned)i, hw_inv) : i; };
    const int c_shift = (C & (C - 1)) == 0 ? 31 - __clz(C) : -1;     // C is a power of two for every bundled network
    // ---- stage x[p][c]
    if (a.p64c4) {
        const bool split = a.p64c4 == kLayoutSplit;
        const uint4* x8 = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(a.x) + (size_t)g * (split ? 8192 : 4096));
        for (int i = t; i < cj * HW; i += kHeadGroup) {
            const int j = i % cj, p = i / cj;
            const int pos = s_pos[p];
            const uint4 v = x8[pos * 8 + (j ^ (pos & 7))];
            const __half2* h2 = reinterpret_cast<const __half2*>(&v);
            float2 f0 = __half22float2(h2[0]), f1 = __half22float2(h2[1]);
            float2 f2 = __half22float2(h2[2]), f3 = __half22float2(h2[3]);
            if (split) {                                   // x = x_h + x_l / 2^11 (second plane)
                const uint4 w = x8[512 + pos * 8 + (j ^ (pos & 7))];
                const __half2* l2 = reinterpret_cast<const __half2*>(&w);
                const float2 g0 = __half22float2(l2[0]), g1 = __half22float2(l2[1]);
                const float2 g2 = __half22float2(l2[2]), g3 = __half22float2(l2[3]);
                f0.x = fmaf(g0.x, kSplitLoUnscale, f0.x); f0.y = fmaf(g0.y, kSplitLoUnscale, f0.y);
                f1.x = fmaf(g1.x, kSplitLoUnscale, f1.x); f1.y = fmaf(g1.y, kSplitLoUnscale, f1.y);
                f2.x = fmaf(g2.x, kSplitLoUnscale, f2.x); f2.y = fmaf(g2.y, kSplitLoUnscale, f2.y);
                f3.x = fmaf(g3.x, kSplitLoUnscale, f3.x); f3.y = fmaf(g3.y, kSplitLoUnscale, f3.y);
            }
            float4* d = reinterpret_cast<float4*>(s_x + p * CP + 8 * j);
            d[0] = make_float4(f0.x, f0.y, f1.x, f1.y);
            d[1] = make_float4(f2.x, f2.y, f3.x, f3.y);
        }
    } else {
        if (tile.src) {
            for (int i = t; i < C * HW; i += kHeadGroup) s_x[tile.xmap[i]] = tile.src[tile.map[i]];
        } else {
            const float* x = a.x + (size_t)g * C * HW;
            for (int i = t; i < C * HW; i += kHeadGroup) { const int c = div_hw(i); s_x[(i - c * HW) * CP + c] = x[i]; }
        }
    }
    group_bar<GROUP>(group);

    if (a.rescaled || a.pool_hidden || a.state_p64c4) {
        // (x - min) / scale per channel over the positions (models.py:530-553).
        // Phase A: channel extrema (two threads per channel when the group is wide enough).
        const int parts = (2 * C <= kHeadGroup) ? 2 : 1;
        for (int i = t; i < parts * C; i += kHeadGroup) {
            const int c = c_shift >= 0 ? (i & (C - 1)) : i % C, part = c_shift >= 0 ? (i >> c_shift) : i / C;
            const int p0 = (part * HW) / parts, p1 = ((part + 1) * HW) / parts;
            float lo = INFINITY, hi = -INFINITY;
            for (int p = p0; p < p1; ++p) { const float v = s_x[p * CP + c]; lo = fminf(lo, v); hi = fmaxf(hi, v); }
            s_part[(part * 2) * C + c] = lo;
            s_part[(part * 2 + 1) * C + c] = hi;
        }
        group_bar<GROUP>(group);
        for (int c = t; c < C; c += kHeadGroup) {
            float lo = s_part[c], hi = s_part[C + c];
            if (parts == 2) { lo = fminf(lo, s_part[2 * C + c]); hi = fmaxf(hi, s_part[3 * C + c]); }
            float sc = __fsub_rn(hi, lo);
            if (sc < 1e-5f) sc = __fadd_rn(sc, 1e-5f);
            s_lo[c] = lo; s_sc[c] = sc;
        }
        group_bar<GROUP>(group);
        // Phase B: normalise and store
        if (a.p64c4) {
            for (int i = t; i < cj * HW; i += kHeadGroup) {
                const int j = i % cj, p = i / cj;
                const int pos = s_pos[p];
                const float4* xr = reinterpret_cast<const float4*>(s_x + p * CP + 8 * j);
                const float4* lr = reinterpret_cast<const float4*>(s_lo + 8 * j);
                const float4* sr = reinterpret_cast<const float4*>(s_sc + 8 * j);
                float v[8];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const float4 x4 = xr[q], l4 = lr[q], c4 = sr[q];
                    v[4 * q + 0] = div_pos_or_zero(__fsub_rn(x4.x, l4.x), c4.x);
                    v[4 * q + 1] = div_pos_or_zero(__fsub_rn(x4.y, l4.y), c4.y);
                    v[4 * q + 2] = div_pos_or_zero(__fsub_rn(x4.z, l4.z), c4.z);
                    v[4 * q + 3] = div_pos_or_zero(__fsub_rn(x4.w, l4.w), c4.w);
                }
                if (a.rescaled) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) a.rescaled[(size_t)g * C * HW + (8 * j + e) * HW + p] = v[e];
                }
                uint4 packed, packed_lo;                        // 16-bit operands of the tensor-core convs
                __half2* h2 = reinterpret_cast<__half2*>(&packed);
                __half2* l2 = reinterpret_cast<__half2*>(&packed_lo);
#pragma unroll
                for (int e = 0; e < 4; ++e) {                   // values are in [0, 1]: no range concerns
                    h2[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
                    const float2 back = __half22float2(h2[e]);
                    l2[e] = __floats2half2_rn((v[2 * e] - back.x) * kSplitLoScale, (v[2 * e + 1] - back.y) * kSplitLoScale);
                }
                const bool split = a.p64c4 == kLayoutSplit;
                const int off8 = pos * 8 + (j ^ (pos & 7));     // in 16-byte units inside the state's first plane
                const size_t board16 = split ? 1024 : 512;      // 16-byte units per stored state
                if (a.pool_hidden) {
                    uint4* dst = reinterpret_cast<uint4*>(a.pool_hidden) + ((size_t)g * a.pool_stride + out_slot) * board16;
                    dst[off8] = packed;
                    if (split) dst[512 + off8] = packed_lo;
                }
                if (a.state_p64c4) {
                    uint4* dst = reinterpret_cast<uint4*>(a.state_p64c4) + (size_t)g * board16;
                    dst[off8] = packed;
                    if (split) dst[512 + off8] = packed_lo;
                }
            }
        } else {
            for (int i = t; i < C * HW; i += kHeadGroup) {
                const int c = div_hw(i), p = i - c * HW;
                const float v = div_pos_or_zero(__fsub_rn(s_x[p * CP + c], s_lo[c]), s_sc[c]);
                if (a.rescaled) a.rescaled[(size_t)g * C * HW + i] = v;
                if (a.pool_hidden) a.pool_hidden[((size_t)g * a.pool_stride + out_slot) * C * HW + i] = v;
                if (tile.dst) tile.dst[tile.map[i]] = v;
            }
        }
    }

    if (a.n_heads > 0) {
        // the heads of this launch side by side: head h owns threads [h*span, (h+1)*span)
        const int span = kHeadGroup / a.n_heads;
        const int h = t / span, u = t % span;
        const HeadDesc& d = a.head[h];
        float* cur = s_act + (size_t)h * 2 * a.smem_floats;
        float* nxt = cur + a.smem_floats;
        // conv1x1: r[c][p] = b[c] + sum_k W[c][k] x[p][k]; one item = (position, group of 4 channels), items spread over the
        // head's threads (a small board with many reduced channels - TicTacToe: 9 positions x 16 channels - keeps every lane
        // busy that way; Connect4's 2-4 reduced channels are one group: one thread per position as before)
        const int n_cgroups = (d.rc + 3) >> 2;
        for (int it = u; it < HW * n_cgroups; it += span) {
            const int cg = div_hw(it), p = it - cg * HW, c0 = cg << 2;
            const float4* xr = reinterpret_cast<const float4*>(s_x + p * CP);
            const int nc = min(4, d.rc - c0);
            float acc[4];
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) acc[cc] = cc < nc ? blob[d.b1_off + c0 + cc] : 0.0f;
            const float4* w0 = reinterpret_cast<const float4*>(blob + d.w1_off + (size_t)c0 * C);
#pragma unroll 4
            for (int k4 = 0; k4 < C / 4; ++k4) {
                const float4 x4 = xr[k4];
#pragma unroll
                for (int cc = 0; cc < 4; ++cc) {
                    if (cc < nc) {
                        const float4 w4 = w0[cc * (C / 4) + k4];
                        acc[cc] = fmaf(w4.x, x4.x, acc[cc]);
                        acc[cc] = fmaf(w4.y, x4.y, acc[cc]);
                        acc[cc] = fmaf(w4.z, x4.z, acc[cc]);
                        acc[cc] = fmaf(w4.w, x4.w, acc[cc]);
                    }
                }
            }
#pragma unroll
            for (int cc = 0; cc < 4; ++cc)
                if (cc < nc) cur[(c0 + cc) * HW + p] = acc[cc];          // flatten order (c, h, w) = NCHW view(-1, ...)
        }
        if (u < 4) { const int i = d.rc * HW + u; if (i < ((d.rc * HW + 3) & ~3)) cur[i] = 0.0f; }   // zero the padding
        group_bar<GROUP>(group);
        const int max_layers = max(a.head[0].mlp.n, a.head[a.n_heads - 1].mlp.n);
        for (int l = 0; l < max_layers; ++l) {
            if (l < d.mlp.n) {
                const int in4 = (d.mlp.in[l] + 3) >> 2, out = d.mlp.out[l];
                const float4* W4 = reinterpret_cast<const float4*>(blob + d.mlp.w_off[l]);      // [in/4][out][4]
                const float4* a4 = reinterpret_cast<const float4*>(cur);
                const float* b = blob + d.mlp.b_off[l];
                const bool last = l == d.mlp.n - 1;
                const int out4 = (out + 3) & ~3;
                // one warp per sample (GROUP == 32): a long dot product with few outputs (TicTacToe's 144 -> 8) would keep 8
                // lanes busy for 36 steps; K is split over `ks` adjacent lanes instead (strided partial sums, a shuffle
                // tree, then the bias).  A different summation order than the one-lane loop - both are fp32 sums compared
                // with the reference under the tolerance of tests/test_resnet_gpu.py.
                int ks = 1;
                if constexpr (GROUP == 32) {
                    while (ks < 8 && 2 * ks * out4 <= span && in4 >= 16 * ks) ks <<= 1;
                }
                if (ks > 1) {
                    const int o = u / ks, part = u % ks;             // out4 * ks <= span: every thread of the head has a slot
                    float acc = 0.0f;
                    if (o < out) {
#pragma unroll 4
                        for (int i = part; i < in4; i += ks) {
                            const float4 x4 = a4[i], w4 = W4[(size_t)i * out + o];
                            acc = fmaf(x4.x, w4.x, acc);
                            acc = fmaf(x4.y, w4.y, acc);
                            acc = fmaf(x4.z, w4.z, acc);
                            acc = fmaf(x4.w, w4.w, acc);
                        }
                    }
                    const unsigned hmask = span >= 32 ? 0xffffffffu : (((1u << span) - 1u) << (h * span));
                    for (int off = ks >> 1; off > 0; off >>= 1) acc += __shfl_xor_sync(hmask, acc, off);
                    if (part == 0 && o < out4) {
                        const float r = acc + (o < out ? b[o] : 0.0f);
                        nxt[o] = o < out ? (last ? r : elu1(r)) : 0.0f;
                    }
                } else {
                    for (int o = u; o < out4; o += span) {
                        if (o < out) {
                            float acc = b[o];
#pragma unroll 4
                            for (int i = 0; i < in4; ++i) {
                                const float4 x4 = a4[i], w4 = W4[(size_t)i * out + o];
                                acc = fmaf(x4.x, w4.x, acc);
                                acc = fmaf(x4.y, w4.y, acc);
                                acc = fmaf(x4.z, w4.z, acc);
                                acc = fmaf(x4.w, w4.w, acc);
                            }
                            nxt[o] = last ? acc : elu1(acc);
                        } else {
                            nxt[o] = 0.0f;                          // padding read by the next layer's float4 loads
                        }
                    }
                }
                float* tmp = cur; cur = nxt; nxt = tmp;
            }
            group_bar<GROUP>(group);
        }
        if (a.logits[h])
            for (int o = u; o < d.n_out; o += span) a.logits[h][(size_t)g * d.n_out + o] = cur[o];
        if (span >= 32) {                              // span is a multiple of 32: the head's first warp
            if (a.scalar[h] && u < 32) {
                const float v = support_to_scalar_group<32>(cur, a.S);
                if (u == 0) a.scalar[h][g] = v;
            }
        } else {
            // two heads share a warp, 16 lanes each: both call the full-mask reduction (common.cuh, LaneGroup); a head
            // without a scalar reduces its first logit only (S = 0) and discards the result
            const float v = support_to_scalar_group<16>(cur, a.scalar[h] ? a.S : 0);
            if (u == 0 && a.scalar[h]) a.scalar[h][g] = v;
        }
    }
    group_bar<GROUP>(group);
}

}  // namespace mz
