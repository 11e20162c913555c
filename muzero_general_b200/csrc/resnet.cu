// Residual MuZero networks (models.py:206-623) on the device - fp32 CUDA-core path.
//
//   representation  models.py:339-349 (+ DownSample models.py:233-275), rescale models.py:526-553
//   dynamics        models.py:379-389, action plane + rescale models.py:555-599
//   prediction      models.py:424-433
//   support_to_scalar models.py:645-666 fused behind the value / reward heads
//
// Layout: activations NCHW fp32 in HBM workspaces; BatchNorm (eval mode, self_play.py:29) is
// folded into the conv weights/bias at load time; the dynamics input plane action/|A|
// (models.py:557-572) is synthesised while staging the input tile, never materialised.
// conv3x3 is a register-tiled direct convolution: a CTA stages the (padded) input planes of
// one or more samples plus the [cin][tap][cout] weights of a cout tile in shared memory; each
// thread owns 4 output channels x P consecutive pixels of one row.
// This is the exact-fp32 path ("strict" numerics, also the validation reference for the
// tensor-core path).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "heads.cuh"
#include "ktimer.h"
#include "small_tower.h"
#include "small_search.h"
#include "launch.h"
#include "conv_tc.h"
#include "conv_wide.h"
#include "cnn_stem.h"
#include "pipeline.h"

namespace mz {

__device__ __forceinline__ float sat_f16_range(float v) { return fminf(fmaxf(v, -65504.0f), 65504.0f); }
__device__ __forceinline__ void split_f32(float v, __half* hi, __half* lo) {
    const __half h = __float2half_rn(sat_f16_range(v));
    *hi = h;
    *lo = __float2half_rn(sat_f16_range((v - __half2float(h)) * kSplitLoScale));
}

// ------------------------------------------------------------------------------------------
// conv3x3 (+folded BN bias, +residual, +ReLU), stride 1 or 2, pad 1
// ------------------------------------------------------------------------------------------
struct ConvArgs {
    const float* in;          // [n, Cin_real, Hin, Win]   (or gathered from the hidden pool)
    float* out;               // [n, Cout, Ho, Wo]
    const float* residual;    // same shape as out or nullptr
    const float* w;           // [Cin][9][Cout]
    const float* bias;        // [Cout] or nullptr
    const int32_t* gather_parent;   // pool mode: sample g reads in + (g*pool_stride + gather_parent[g]) * sample_elems
    const int32_t* action;    // extra constant input plane action/A as channel Cin-1 (dynamics), or nullptr
    int pool_stride;
    int n, Cin, Cout, Hin, Win, Ho, Wo, stride, relu, A;
    int boards_per_cta, cin_chunk;
    int cout_tile;            // output channels per CTA (blockIdx.y picks the tile): 64, or fewer when one row of 64 is too many items
    int band_rows;            // output rows per CTA (blockIdx.z picks the band); = Ho unless the image is too large for one CTA
    int out_p64c4;            // kLayoutF16 / kLayoutSplit: write the tensor-core board layout (P64S) instead of NCHW
};

template <int P, int STRIDE, int MAX_ITEMS>
__global__ void __launch_bounds__(256) conv3x3_kernel(const __grid_constant__ ConvArgs a) {
    extern __shared__ __align__(16) float smem[];
    constexpr int IN_SPAN = (P - 1) * STRIDE + 3;              // input columns feeding P outputs
    // this CTA's band of output rows [r0, r0 + nbr) and the input rows it needs: [r0*STRIDE - 1, (r0+nbr-1)*STRIDE + 1]
    const int r0 = blockIdx.z * a.band_rows;
    const int nbr = min(a.band_rows, a.Ho - r0);
    const int y_in0 = r0 * STRIDE - 1;
    const int Hp = (a.band_rows - 1) * STRIDE + 3, Wp = a.Win + 2;   // staged (padded) plane of the band
    const int plane = Hp * Wp;
    // cout tiles of cout_tile (<= 64) channels; the last one holds the remaining Cout - cout0 (a multiple of 4)
    const int cout0 = blockIdx.y * a.cout_tile;
    const int ct = min(a.Cout - cout0, a.cout_tile);            // cout tile of this CTA
    const int cgs = ct / 4;
    const int segs = a.Wo / P;
    const int items_per_board = cgs * nbr * segs;
    const int b0 = blockIdx.x * a.boards_per_cta;
    const int nb = min(a.boards_per_cta, a.n - b0);
    float* s_w = smem;                                          // [cin_chunk][9][ct]
    float* s_in = smem + a.cin_chunk * 9 * ct;                  // [boards][cin_chunk][Hp][Wp]
    const int cin_real = a.action ? a.Cin - 1 : a.Cin;
    const size_t sample_elems = (size_t)cin_real * a.Hin * a.Win;

    const int total_items = nb * items_per_board;
    // each thread may own several items (big images): MAX_ITEMS accumulator tiles
    float acc[MAX_ITEMS][4][P];
#pragma unroll
    for (int it = 0; it < MAX_ITEMS; ++it)
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int p = 0; p < P; ++p) acc[it][c][p] = 0.0f;

    for (int c0 = 0; c0 < a.Cin; c0 += a.cin_chunk) {
        const int cc = min(a.cin_chunk, a.Cin - c0);
        __syncthreads();
        // ---- stage weights of this cin chunk / cout tile
        // (as float4: Cout, cout0 and ct are multiples of 4 and every layer of the blob starts 16-byte aligned; one
        // integer division per 4 weights instead of per weight matters when a CTA stages 64 x 9 x 64 of them)
        for (int i = threadIdx.x; i < cc * 9 * ct / 4; i += blockDim.x) {
            const int co = (i % (ct / 4)) * 4, r = i / (ct / 4);           // r = ci*9 + tap
            *reinterpret_cast<float4*>(s_w + r * ct + co) =
                *reinterpret_cast<const float4*>(a.w + ((size_t)(c0 * 9 + r)) * a.Cout + cout0 + co);
        }
        // ---- stage padded input planes
        for (int i = threadIdx.x; i < nb * cc * plane; i += blockDim.x) {
            const int x = i % Wp, y = (i / Wp) % Hp, ci = (i / plane) % cc, b = i / (plane * cc);
            const int g = b0 + b, cg = c0 + ci;
            float v = 0.0f;
            const int yi = y_in0 + y;                           // input row of staged row y
            if (x >= 1 && x <= a.Win && yi >= 0 && yi < a.Hin) {
                if (a.action && cg == a.Cin - 1) {
                    v = __fdiv_rn((float)a.action[g], (float)a.A);       // action / |A| plane
                } else {
                    const float* src = a.gather_parent
                        ? a.in + ((size_t)g * a.pool_stride + a.gather_parent[g]) * sample_elems
                        : a.in + (size_t)g * sample_elems;
                    v = src[((size_t)cg * a.Hin + yi) * a.Win + (x - 1)];
                }
            }
            s_in[i] = v;
        }
        __syncthreads();
        // ---- accumulate
#pragma unroll
        for (int it = 0; it < MAX_ITEMS; ++it) {
            const int item = threadIdx.x + it * blockDim.x;
            if (item >= total_items) break;
            const int cgi = item % cgs;
            const int rest = item / cgs;
            const int seg = rest % segs, y = (rest / segs) % nbr, b = rest / (segs * nbr);
            const float* ib = s_in + (size_t)b * cc * plane + (y * STRIDE) * Wp + seg * P * STRIDE;
            const float* wb = s_w + cgi * 4;
            for (int ci = 0; ci < cc; ++ci) {
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    float v[IN_SPAN];
#pragma unroll
                    for (int j = 0; j < IN_SPAN; ++j) v[j] = ib[ci * plane + dy * Wp + j];
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const float4 w4 = *reinterpret_cast<const float4*>(wb + (ci * 9 + dy * 3 + dx) * ct);
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            const float xv = v[p * STRIDE + dx];
                            acc[it][0][p] = fmaf(xv, w4.x, acc[it][0][p]);
                            acc[it][1][p] = fmaf(xv, w4.y, acc[it][1][p]);
                            acc[it][2][p] = fmaf(xv, w4.z, acc[it][2][p]);
                            acc[it][3][p] = fmaf(xv, w4.w, acc[it][3][p]);
                        }
                    }
                }
            }
        }
    }
    // ---- epilogue
#pragma unroll
    for (int it = 0; it < MAX_ITEMS; ++it) {
        const int item = threadIdx.x + it * blockDim.x;
        if (item >= total_items) break;
        const int cgi = item % cgs;
        const int rest = item / cgs;
        const int seg = rest % segs, y = r0 + (rest / segs) % nbr, b = rest / (segs * nbr);
        const int g = b0 + b;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int co = cout0 + cgi * 4 + c;
            const float bias = a.bias ? a.bias[co] : 0.0f;
            const size_t o = (((size_t)g * a.Cout + co) * a.Ho + y) * a.Wo + seg * P;
#pragma unroll
            for (int p = 0; p < P; ++p) {
                float r = acc[it][c][p] + bias;
                if (a.residual) r += a.residual[o + p];
                if (a.relu) r = fmaxf(r, 0.0f);
                if (a.out_p64c4) {
                    const int pos = (y + 1) * 8 + seg * P + p;
                    const int e = pos * 64 + (((co >> 3) ^ (pos & 7)) << 3) + (co & 7);
                    if (a.out_p64c4 == kLayoutSplit) {
                        __half* base = reinterpret_cast<__half*>(a.out) + (size_t)g * 8192;
                        split_f32(r, base + e, base + 4096 + e);
                    } else {
                        reinterpret_cast<__half*>(a.out)[(size_t)g * 4096 + e] = __float2half_rn(r);
                    }
                }
                else
                    a.out[o + p] = r;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// AvgPool2d(kernel 3, stride 2, padding 1), count_include_pad (always / 9)   models.py:258,262
// ------------------------------------------------------------------------------------------
__global__ void avgpool3x3s2_kernel(const float* in, float* out, int planes, int H, int W, int Ho, int Wo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)planes * Ho * Wo) return;
    const int x = i % Wo, y = (i / Wo) % Ho;
    const size_t pl = i / ((size_t)Wo * Ho);
    const float* p = in + pl * H * W;
    float s = 0.0f;
    for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
            const int yy = 2 * y + dy, xx = 2 * x + dx;
            if (yy >= 0 && yy < H && xx >= 0 && xx < W) s += p[yy * W + xx];
        }
    out[i] = __fdiv_rn(s, 9.0f);
}

template <int GROUP>
__global__ void __launch_bounds__(kHeadThreads) heads_kernel(const __grid_constant__ HeadsArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int group = threadIdx.x / GROUP, t = threadIdx.x % GROUP, ngroups = blockDim.x / GROUP;
    float* s_w = sm;                                                 // head blob slice [w_lo, w_lo + w_floats)
    float* scratch = s_w + a.w_floats + (size_t)group * a.warp_floats;
    // board layout only (C = 64): padded row of dense position p, looked up instead of two runtime divisions per chunk
    __shared__ unsigned char s_pos[64];
    pdl_launch_dependents();
    {
        const float4* src = reinterpret_cast<const float4*>(a.blob + a.w_lo);
        float4* dst = reinterpret_cast<float4*>(s_w);
        for (int i = threadIdx.x; i < a.w_floats / 4; i += blockDim.x) dst[i] = src[i];
        if (a.p64c4 && threadIdx.x < a.HW && threadIdx.x < 64)
            s_pos[threadIdx.x] = (unsigned char)((threadIdx.x / a.W + 1) * 8 + (threadIdx.x % a.W));
    }
    __syncthreads();
    pdl_wait();                                                      // the weights are constants; x comes from the previous kernel
    const float* blob = s_w - a.w_lo;                                // blob[off] addresses the staged copy
    for (int g = a.g0 + blockIdx.x * ngroups + group; g < a.g0 + a.n; g += gridDim.x * ngroups)
        heads_one_sample<GROUP>(a, blob, scratch, s_pos, g, group, t, a.out_slot);
}

// ------------------------------------------------------------------------------------------
// Generic heads for nets whose head weights do not fit in shared memory (games/atari.py: 256 reduced channels x 36
// positions -> FC 9216 -> 256 -> 256 -> 601, 9.4 MB for the first FC layer alone): the same operations as heads_kernel,
// one plain kernel per stage, every dot product accumulated in ascending order from the bias.  The two routes agree bit
// for bit on the rescaled state always; on the logits of a layer where heads_kernel adds with one lane per output
// (heads_kernel<128>, and heads_kernel<32> where the split-K width ks is 1); on the scalar where heads_kernel reduces it
// with 32 lanes (heads_kernel<128>, and heads_kernel<32> with one head per warp) - not where two heads share a warp, 16
// lanes each (tests/test_heads_gpu.py::test_forced_routes_agree).  Throughput is not the point here - availability of the
// large configuration is.
// ------------------------------------------------------------------------------------------
__global__ void big_rescale_kernel(const float* x, int n, int C, int HW, float* rescaled, float* pool_hidden, int pool_stride, int out_slot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;           // (sample, channel)
    if (i >= n * C) return;
    const int g = i / C;
    const float* src = x + (size_t)i * HW;
    float lo = INFINITY, hi = -INFINITY;
    for (int p = 0; p < HW; ++p) { lo = fminf(lo, src[p]); hi = fmaxf(hi, src[p]); }
    float sc = __fsub_rn(hi, lo);
    if (sc < 1e-5f) sc = __fadd_rn(sc, 1e-5f);
    for (int p = 0; p < HW; ++p) {
        const float v = div_pos_or_zero(__fsub_rn(src[p], lo), sc);
        if (rescaled) rescaled[(size_t)i * HW + p] = v;
        if (pool_hidden) pool_hidden[((size_t)g * pool_stride + out_slot) * C * HW + (size_t)(i % C) * HW + p] = v;
    }
}
// r[g][c][p] = b[c] + sum_k W[c][k] x[g][k][p]
__global__ void big_conv1x1_kernel(const float* x, const float* w, const float* b, int n, int C, int rc, int HW, float* out, int out_stride) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * rc * HW) return;
    const int p = i % HW, c = (i / HW) % rc;
    const size_t g = i / ((size_t)HW * rc);
    const float* xs = x + g * C * HW + p;
    const float* ws = w + (size_t)c * C;
    float acc = b[c];
    for (int k = 0; k < C; ++k) acc = fmaf(ws[k], xs[(size_t)k * HW], acc);
    out[g * out_stride + (size_t)c * HW + p] = acc;
}
// y[g][o] = act(b[o] + sum_i x[g][i] W[i][o]), W packed [in/4][out][4]; x rows are `in_stride` apart and zero padded to 4
__global__ void big_fc_kernel(const float* x, const float* W, const float* b, int n, int in, int out, int in_stride, int out_stride,
                              int elu, float* y) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int out4 = (out + 3) & ~3;
    if (i >= (size_t)n * out4) return;
    const int o = i % out4;
    const size_t g = i / out4;
    float r = 0.0f;
    if (o < out) {
        const float4* x4 = reinterpret_cast<const float4*>(x + g * in_stride);
        const float4* W4 = reinterpret_cast<const float4*>(W);
        float acc = b[o];
        const int in4 = (in + 3) >> 2;
        for (int k = 0; k < in4; ++k) {
            const float4 xv = x4[k], wv = W4[(size_t)k * out + o];
            acc = fmaf(xv.x, wv.x, acc);
            acc = fmaf(xv.y, wv.y, acc);
            acc = fmaf(xv.z, wv.z, acc);
            acc = fmaf(xv.w, wv.w, acc);
        }
        r = elu ? elu1(acc) : acc;
    }
    y[g * out_stride + o] = r;                                     // the padding entries read by the next layer are zero
}
__global__ void big_scalar_kernel(const float* logits, int n, int stride, int n_out, int S, float* logits_out, float* scalar) {
    const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= n) return;
    const float* l = logits + (size_t)g * stride;
    if (logits_out) for (int o = lane; o < n_out; o += 32) logits_out[(size_t)g * n_out + o] = l[o];
    if (scalar) {
        const float v = support_to_scalar_group<32>(l, S);
        if (lane == 0) scalar[g] = v;
    }
}

__global__ void fill_root_reward_logits_kernel(float* out, int n, int F, int S) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * F) out[i] = (i % F == S) ? 0.0f : -INFINITY;
}
__global__ void fill_root_reward_kernel(float* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = inverse_value_transform(0.0f);
}
__global__ void copy_from_pool_kernel(const float* pool, float* out, int n, int pool_stride, int slot, int elems) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * elems) return;
    const size_t g = i / elems, e = i % elems;
    out[i] = pool[(g * pool_stride + slot) * elems + e];
}

// dense fp32 NCHW [count][C][H*W]  <->  fp16 P64C8 [count][C/8][64][8]
__global__ void nchw_to_p64c4_kernel(const float* in, float* out, int count, int C, int H, int W, int split) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int HW = H * W;
    if (i >= (size_t)count * C * HW) return;
    const size_t g = i / ((size_t)C * HW);
    const int c = (i / HW) % C, p = i % HW;
    const int e = p64c4_index(c, p, W);
    if (split) {
        __half* base = reinterpret_cast<__half*>(out) + g * 8192;
        split_f32(in[i], base + e, base + 4096 + e);
    } else {
        reinterpret_cast<__half*>(out)[g * 4096 + e] = __float2half_rn(in[i]);
    }
}
__global__ void p64c4_to_nchw_kernel(const float* in, float* out, int count, int C, int H, int W, int split) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int HW = H * W;
    if (i >= (size_t)count * C * HW) return;
    const size_t g = i / ((size_t)C * HW);
    const int c = (i / HW) % C, p = i % HW;
    const int e = p64c4_index(c, p, W);
    if (split) {
        const __half* base = reinterpret_cast<const __half*>(in) + g * 8192;
        out[i] = fmaf(__half2float(base[4096 + e]), kSplitLoUnscale, __half2float(base[e]));
    } else {
        out[i] = __half2float(reinterpret_cast<const __half*>(in)[g * 4096 + e]);
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
struct ConvLayer {
    int cin, cout, stride;
    size_t w_off;             // into the conv blob: [cin][9][cout]
    long b_off;               // folded BN bias [cout], -1 = none
    long tc_off;              // tensor-core image [9][C/4][C][4] (tf32), or the wide towers' x3 image (conv_wide.h), -1 = none
    long tc_table_off;        // dynamics first conv: action-plane table [64][C] ([H * W][C] on the wide towers), -1 = none
    long tc_scale_off;        // x3 mode: [C] per-output-channel power of two undoing the weight prescale, -1 = none
};

struct ResNetDevice {
    MzNetDesc net;
    int max_batch, sm_count;
    int C, hh, hw;            // hidden state geometry
    // layers in execution order
    std::vector<ConvLayer> rep_down;   // conv1, rb1 x2 (2 convs each), conv2, rb2 x3, rb3 x3   (downsample only)
    std::vector<ConvLayer> rep_trunk;  // [stem conv if no downsample] + blocks x 2
    CnnStemWeights cnn{};              // downsample = 2: DownsampleCNN's two convs in the conv blob (cnn_stem.cu)
    std::vector<ConvLayer> dyn;        // conv + blocks x 2
    std::vector<ConvLayer> pred;       // blocks x 2
    HeadDesc reward_head, value_head, policy_head;
    float* d_conv = nullptr;           // conv weights + biases
    float* d_head = nullptr;           // head blob
    float* ws[3] = {nullptr, nullptr, nullptr};
    size_t ws_elems = 0;
    float* scratch_hidden = nullptr;   // [B, C*hh*hw] rescaled state when no pool is given (dense NCHW)
    float* scratch_state = nullptr;    // [B, 4096 fp16] same state in P64C8 (tensor-core path)
    bool loaded = false;
    TowerRoute route = TowerRoute::CudaCore;
    std::string note;                  // CudaCore only: mz_numerics when a tensor-core route was wanted and not taken, or left
    float* big_scratch = nullptr;      // activations of the generic heads route (heads_big)
    size_t big_elems = 0;
    int* d_sat = nullptr;              // x3 mode: number of epilogue threads that stored an activation beyond the fp16 range
    bool fuse_small = true;            // CUDA-core towers as one fused launch where they fit (small_tower.cu); MZ_NO_FUSE=1: per layer
};

static bool is_tc(TowerRoute t) { return t == TowerRoute::TcF16 || t == TowerRoute::TcX3; }
static bool is_wide(TowerRoute t) { return t == TowerRoute::Wide || t == TowerRoute::WidePair || t == TowerRoute::Wide256; }
// layout of the stored hidden states and of the tensor-core towers' workspaces
static int state_layout(TowerRoute t) {
    return t == TowerRoute::TcX3 ? kLayoutSplit : t == TowerRoute::TcF16 ? kLayoutF16 : kLayoutDense;
}
// the x3 range guard counts saturated activations on these routes (conv_x3.cu, conv_wide.cu, conv_wide256.cu)
static bool range_guarded(TowerRoute t) { return t == TowerRoute::TcX3 || is_wide(t); }
// float slots per stored hidden state: dense C*H*W, or a board of the tensor-core layout (2048 or 4096)
static int state_elems(const ResNetDevice* r) {
    return is_tc(r->route) ? conv_tc_board_elems(r->route == TowerRoute::TcX3) : r->C * r->hh * r->hw;
}

static int conv_out(int h, int stride) { return (h - 1) / stride + 1; }

// Launch plan of one conv3x3_kernel call: n boards of cin x H x W -> cout x Ho x Wo.  The launcher (Runner::conv),
// resnet_create's check of every conv layer of a net and mz_debug_conv3x3_plan all take it from conv3x3_plan.
struct ConvPlan {
    int P, stride, max_items;      // template arguments: pixels per thread, stride, accumulator tiles per thread (1 or 4)
    int bands, band_rows;          // output rows split into bands of band_rows rows (the last one may be shorter)
    int boards, cin_chunk;         // boards per CTA (the last CTA may hold fewer), input channels staged at a time
    int cout_tile;                 // output channels per CTA (the last tile may hold fewer): 64 unless a row of 64 does not fit
    dim3 grid;                     // (board groups, cout tiles, bands)
    size_t smem;                   // dynamic shared memory bytes
};
constexpr int kConvThreads = 256;

// false (with the reason in *err) when the shape cannot be launched
static bool conv3x3_plan(int n, int cin, int cout, int Hin, int Win, int stride, ConvPlan* p, std::string* err) {
    if (n < 1 || cin < 1 || Hin < 1 || Win < 1) { *err = "conv3x3: empty shape"; return false; }
    if (cout < 4 || cout % 4 != 0) { *err = "conv3x3: cout must be a positive multiple of 4"; return false; }
    if (stride != 1 && stride != 2) { *err = "conv3x3: stride must be 1 or 2"; return false; }
    const int Ho = conv_out(Hin, stride), Wo = conv_out(Win, stride);
    p->stride = stride;
    p->P = 1;
    for (int cand : {8, 7, 6, 4, 3, 2}) if (Wo % cand == 0) { p->P = cand; break; }
    const int threads = kConvThreads;
    int ct = cout < 64 ? cout : 64;                // the widest cout tile sizes the items and the weight slice
    // One output row of a 64-channel tile may exceed the item budget on its own (P = 1 on a board more than 64 wide, e.g.
    // DownSample's first convs at 128 channels on a 129-wide frame): halve the tile until a row fits.  Every shape whose
    // row fits keeps the 64-channel tile and the plan it always had.
    while (ct > 4 && (ct / 4) * (Wo / p->P) > threads * 4) ct = (ct / 2 + 3) / 4 * 4;
    p->cout_tile = ct;
    // large images (e.g. 128 output channels at 48 x 48, games/atari.py): split the output rows into bands, one CTA each
    int bands = 1;
    while (bands < Ho && (ct / 4) * ((Ho + bands - 1) / bands) * (Wo / p->P) > threads * 4) ++bands;
    p->band_rows = (Ho + bands - 1) / bands;
    p->bands = (Ho + p->band_rows - 1) / p->band_rows;
    const int items_per_board = (ct / 4) * p->band_rows * (Wo / p->P);
    int boards = 1;
    if (items_per_board < threads) boards = threads / items_per_board;
    if (boards > 32) boards = 32;
    if (boards > n) boards = n;
    if (items_per_board * boards > threads * 4) { *err = "conv3x3: image too large for the item budget"; return false; }
    const size_t plane = (size_t)((p->band_rows - 1) * stride + 3) * (Win + 2);
    // pick the cin chunk so weights + planes fit comfortably
    const size_t budget = 200 * 1024 / 4;
    int chunk = cin;
    while (chunk > 1 && (size_t)chunk * 9 * ct + (size_t)boards * chunk * plane > budget) chunk = (chunk + 1) / 2;
    if ((size_t)chunk * 9 * ct + (size_t)boards * chunk * plane > budget) { *err = "conv3x3: tile does not fit in shared memory"; return false; }
    p->boards = boards; p->cin_chunk = chunk;
    p->max_items = items_per_board * boards > threads ? 4 : 1;
    p->smem = ((size_t)chunk * 9 * ct + (size_t)boards * chunk * plane) * 4;
    p->grid = dim3((n + boards - 1) / boards, (cout + ct - 1) / ct, p->bands);
    return true;
}

// The distinct conv shapes of a net's stage, named for the refusal message
struct ConvShape { const char* stage; int cin, cout, H, W, stride; };
static std::vector<ConvShape> downsample_shapes(int obs_c, int C, int H, int W) {
    const int h1 = conv_out(H, 2), w1 = conv_out(W, 2), h2 = conv_out(h1, 2), w2 = conv_out(w1, 2);
    return {{"DownSample conv1", obs_c, C / 2, H, W, 2}, {"DownSample resblocks1", C / 2, C / 2, h1, w1, 1},
            {"DownSample conv2", C / 2, C, h1, w1, 2}, {"DownSample resblocks2", C, C, h2, w2, 1},
            {"DownSample resblocks3", C, C, conv_out(h2, 2), conv_out(w2, 2), 1}};
}
// false with the first refused shape's reason and stage in *err
static bool plan_shapes(int n, const std::vector<ConvShape>& shapes, std::string* err) {
    for (const ConvShape& s : shapes) {
        ConvPlan p;
        std::string why;
        if (!conv3x3_plan(n, s.cin, s.cout, s.H, s.W, s.stride, &p, &why)) {
            *err = why + " (" + s.stage + ": " + std::to_string(s.cin) + " -> " + std::to_string(s.cout) + " channels, stride " +
                   std::to_string(s.stride) + ", " + std::to_string(s.H) + " x " + std::to_string(s.W) + " input)";
            return false;
        }
    }
    return true;
}

// Offsets of one head in the head blob, which holds *size floats so far: conv1x1 weight [rc][C] and bias [rc], then per
// FC layer the weights packed [in/4][out][4] (zero rows pad `in`) and the bias; every part that is read as float4 starts
// 16-byte aligned.  *size grows by the head.
static void layout_head(int C, int rc, int HW, const int32_t* hidden, int n_hidden, int n_out, size_t* size, HeadDesc& d) {
    size_t o = (*size + 3) & ~(size_t)3;
    d.rc = rc; d.n_out = n_out;
    d.w1_off = (int)o; o += (size_t)rc * C;
    d.b1_off = (int)o; o += rc;
    int sz[MZ_MAX_LAYERS + 2];
    sz[0] = rc * HW;
    for (int i = 0; i < n_hidden; ++i) sz[i + 1] = hidden[i];
    sz[n_hidden + 1] = n_out;
    d.mlp.n = n_hidden + 1;
    for (int l = 0; l < d.mlp.n; ++l) {
        const int in = sz[l], out = sz[l + 1];
        d.mlp.in[l] = in; d.mlp.out[l] = out;
        o = (o + 3) & ~(size_t)3;
        d.mlp.w_off[l] = (int)o; o += (size_t)((in + 3) / 4) * out * 4;
        d.mlp.b_off[l] = (int)o; o += out;
    }
    *size = (o + 3) & ~(size_t)3;
}

// Shared memory of one heads_kernel launch over the heads hs[0, n_heads): the slice [w_lo, w_lo + w_floats) of the head
// blob covering them, and per group of threads an x tile + channel stats + (ping, pong) rows as wide as the widest layer.
struct HeadsFootprint { int w_lo, w_floats, smem_floats, warp_floats; };
static HeadsFootprint heads_footprint(int C, int HW, int n_heads, const HeadDesc* const* hs) {
    int maxw = 32, lo = 1 << 30, hi = 0;
    for (int i = 0; i < n_heads; ++i) {
        const HeadDesc& d = *hs[i];
        maxw = std::max(maxw, d.rc * HW + 4);
        for (int l = 0; l < d.mlp.n; ++l) maxw = std::max(maxw, d.mlp.out[l] + 4);
        lo = std::min(lo, d.w1_off);
        hi = std::max(hi, d.mlp.b_off[d.mlp.n - 1] + d.mlp.out[d.mlp.n - 1]);
    }
    if (n_heads == 0) { lo = 0; hi = 0; }
    HeadsFootprint f;
    f.w_lo = lo; f.w_floats = ((hi - lo) + 3) & ~3;
    f.smem_floats = (maxw + 3) & ~3;
    f.warp_floats = (HW * (C + 4) + 6 * C + 4 * f.smem_floats + 3) & ~3;
    return f;
}
static bool heads_fit_one_group(const HeadsFootprint& f) { return ((size_t)f.w_floats + f.warp_floats) * 4 <= 227 * 1024; }

// The tower route of a net at max_batch boards, from its shape and MZ_TC_MODE / MZ_NO_TC / MZ_TC_WIDE; *note as
// ResNetDevice::note.  Allocates nothing.
static TowerRoute choose_route(const MzNetDesc& net, int hh, int hw, int max_batch, int sm_count, std::string* note) {
    // MZ_TC_MODE = "off": fp32 CUDA-core towers everywhere; anything else: tensor-core towers where the shape allows
    // (conv_tc.cu).  MZ_NO_TC=1 is the older spelling of "off".
    const char* no_tc = getenv("MZ_NO_TC");
    const char* tc_mode = getenv("MZ_TC_MODE");
    if ((no_tc && no_tc[0] == '1') || (tc_mode && strcmp(tc_mode, "off") == 0)) return TowerRoute::CudaCore;
    // default "x3": split 16-bit operands, three partial products, fp32-grade accuracy; "fp16": plain fp16 operands
    // (3x fewer MMAs, ~1e-2 hidden-state error: opt-in)
    const bool fp16 = tc_mode && strcmp(tc_mode, "fp16") == 0;
    if (!net.downsample && conv_tc_supported(net.channels, net.obs_h, net.obs_w)) {
        // The heads of the tensor-core route read the board layout and have no generic (global-memory) variant.  A net
        // whose head weights do not fit in shared memory next to one sample's tile (e.g. support 300, or a 128-wide value
        // layer over 16 reduced channels) runs on the fp32 CUDA-core towers and the generic heads route instead.
        const int C = net.channels, HW = net.obs_h * net.obs_w, F = 2 * net.support_size + 1;
        HeadDesc reward, value, policy;
        size_t size = 0;
        layout_head(C, net.reduced_reward, HW, net.res_fc_reward, net.n_res_fc_reward, F, &size, reward);
        layout_head(C, net.reduced_value, HW, net.res_fc_value, net.n_res_fc_value, F, &size, value);
        layout_head(C, net.reduced_policy, HW, net.res_fc_policy, net.n_res_fc_policy, net.action_space, &size, policy);
        const HeadDesc* calls[3][2] = {{nullptr, nullptr}, {&reward, nullptr}, {&value, &policy}};
        for (int n_heads = 0; n_heads < 3; ++n_heads)
            if (!heads_fit_one_group(heads_footprint(C, HW, n_heads, calls[n_heads]))) {
                *note = "f32 nets + f64 tree statistics (no tensor-core towers: the head weights exceed shared memory)";
                return TowerRoute::CudaCore;
            }
        return fp16 ? TowerRoute::TcF16 : TowerRoute::TcX3;
    }
    // MZ_TC_WIDE=1 (opt-in until measured): the towers of a 128-channel net as x3 tensor-core launches on the dense states
    // (conv_wide.cu), when the planner accepts the hidden board.  The stems and the heads stay on the CUDA cores.
    // MZ_TC_WIDE=2: the same, and a board the one-CTA plan refuses (15 x 15, 16 x 16) is split across CTA pairs.
    // MZ_TC_WIDE=3: as 2, and the towers of a 256-channel net (games/atari.py) on the hidden board hh x hw, with any
    // representation stem, as x3 tensor-core launches with the output channels split across CTA pairs (conv_wide256.cu).
    const char* wide_env = getenv("MZ_TC_WIDE");
    if (wide_env && wide_env[0] == '3' && !fp16 && net.channels == kWide256C) {
        Wide256Plan p;
        const char* why = "";
        if (wide256_plan(max_batch, net.channels, hh, hw, 1 + 2 * net.blocks, sm_count, 0, &p, &why)) return TowerRoute::Wide256;
        *note = std::string("f32 nets + f64 tree statistics (256-channel towers stay on the CUDA cores: ") + why + ")";
        return TowerRoute::CudaCore;
    }
    if (!wide_env || (wide_env[0] != '1' && wide_env[0] != '2' && wide_env[0] != '3') || fp16 || net.channels != kWideC ||
        net.downsample)
        return TowerRoute::CudaCore;
    const int layers = 1 + 2 * net.blocks;
    WideTowerPlan p;
    const char* why = "";
    if (wide_tower_plan(max_batch, net.channels, net.obs_h, net.obs_w, layers, sm_count, &p, &why)) return TowerRoute::Wide;
    std::string reasons = why;
    if (wide_env[0] != '1') {
        const char* why_pair = "";
        if (wide_pair_plan(max_batch, net.channels, net.obs_h, net.obs_w, layers, sm_count, &p, &why_pair)) return TowerRoute::WidePair;
        reasons = std::string("one CTA: ") + why + "; CTA pairs: " + why_pair;
    }
    *note = "f32 nets + f64 tree statistics (128-channel towers stay on the CUDA cores: " + reasons + ")";
    return TowerRoute::CudaCore;
}

ResNetDevice* resnet_create(const MzNetDesc& net, int max_batch, int sm_count, std::string* err) {
    ResNetDevice* r = new ResNetDevice();
    r->net = net; r->max_batch = max_batch; r->sm_count = sm_count;
    r->C = net.channels;
    if (net.channels % 4 != 0 || (net.downsample == 1 && (net.channels / 2) % 4 != 0)) {
        *err = "channels must be a multiple of 4 (8 with downsample=\"resnet\")";
        delete r; return nullptr;
    }
    int H = net.obs_h, W = net.obs_w;
    size_t max_elems = (size_t)net.obs_c * H * W;
    if (net.downsample == 2) {
        // DownsampleCNN: every geometry the reference's module cannot run is refused here, naming the stage
        CnnStemPlan p;
        std::string why;
        if (!cnn_stem_plan(max_batch, net.obs_c, net.channels, H, W, sm_count, &p, &why)) {
            *err = "downsample=\"CNN\" (" + std::to_string(net.obs_c) + " x " + std::to_string(H) + " x " + std::to_string(W) +
                   " observation): " + why;
            delete r; return nullptr;
        }
        r->hh = p.h; r->hw = p.w;
        max_elems = std::max(max_elems, (size_t)p.mid * p.s[0].Hp * p.s[0].Wp);
        max_elems = std::max(max_elems, (size_t)net.channels * p.h * p.w);
    } else if (net.downsample) {
        int h1 = conv_out(H, 2), w1 = conv_out(W, 2);
        int h2 = conv_out(h1, 2), w2 = conv_out(w1, 2);
        int h3 = conv_out(h2, 2), w3 = conv_out(w2, 2);
        int h4 = conv_out(h3, 2), w4 = conv_out(w3, 2);
        max_elems = std::max(max_elems, (size_t)(net.channels / 2) * h1 * w1);
        max_elems = std::max(max_elems, (size_t)net.channels * h2 * w2);
        r->hh = h4; r->hw = w4;
        if (h4 != (H + 15) / 16 || w4 != (W + 15) / 16) {
            *err = "downsample geometry does not match ceil(H/16) x ceil(W/16) (models.py:456-484)";
            delete r; return nullptr;
        }
    } else {
        r->hh = H; r->hw = W;
        max_elems = std::max(max_elems, (size_t)net.channels * H * W);
    }
    max_elems = std::max(max_elems, (size_t)(net.channels + 1) * r->hh * r->hw);
    // Every conv of the net must have a conv3x3_kernel launch plan (it is the route of the stems and the fallback of
    // every other tower), so a shape the planner refuses fails here, not part-way through a search.  A plan that exists
    // for max_batch boards exists for any smaller batch (fewer boards per CTA only shrink the tile).
    {
        const int C = net.channels, h = r->hh, w = r->hw;
        std::vector<ConvShape> shapes;
        if (net.downsample == 1) {
            shapes = downsample_shapes(net.obs_c, C, H, W);
        } else if (net.downsample == 2) {
            // the stem was planned above; the representation trunk is blocks only
        } else {
            shapes = {{"representation stem", net.obs_c, C, H, W, 1}};
        }
        shapes.push_back({"dynamics stem", C + 1, C, h, w, 1});                     // (action plane)
        if (net.blocks > 0) shapes.push_back({"residual blocks", C, C, h, w, 1});
        if (!plan_shapes(max_batch, shapes, err)) { delete r; return nullptr; }
    }
    // the route is known here, so the hidden-state pool and the workspaces are sized for it
    r->route = choose_route(net, r->hh, r->hw, max_batch, sm_count, &r->note);
    const char* no_fuse = getenv("MZ_NO_FUSE");
    r->fuse_small = !(no_fuse && no_fuse[0] == '1');
    max_elems = std::max(max_elems, (size_t)state_elems(r));
    r->ws_elems = max_elems * (size_t)max_batch;
    for (int i = 0; i < 3; ++i) {
        if (cudaMalloc(&r->ws[i], r->ws_elems * 4 + 64) != cudaSuccess) { *err = "workspace allocation failed"; resnet_destroy(r); return nullptr; }
        cudaMemset(r->ws[i], 0, r->ws_elems * 4 + 64);      // P64C4 padding positions must read as zero
    }
    if (cudaMalloc(&r->scratch_hidden, (size_t)max_batch * r->C * r->hh * r->hw * 4 + 64) != cudaSuccess ||
        cudaMalloc(&r->scratch_state, (size_t)max_batch * state_elems(r) * 4 + 64) != cudaSuccess) {
        *err = "workspace allocation failed"; resnet_destroy(r); return nullptr;
    }
    cudaMemset(r->scratch_state, 0, (size_t)max_batch * state_elems(r) * 4 + 64);
    if (cudaMalloc(&r->d_sat, 64) != cudaSuccess) { *err = "workspace allocation failed"; resnet_destroy(r); return nullptr; }
    cudaMemset(r->d_sat, 0, 64);
    return r;
}

void resnet_destroy(ResNetDevice* r) {
    if (!r) return;
    for (int i = 0; i < 3; ++i) if (r->ws[i]) cudaFree(r->ws[i]);
    if (r->scratch_hidden) cudaFree(r->scratch_hidden);
    if (r->scratch_state) cudaFree(r->scratch_state);
    if (r->d_sat) cudaFree(r->d_sat);
    if (r->big_scratch) cudaFree(r->big_scratch);
    if (r->d_conv) cudaFree(r->d_conv);
    if (r->d_head) cudaFree(r->d_head);
    delete r;
}

namespace {
struct Loader {
    const MzTensor* t; int n; std::string* err; bool ok = true;
    const MzTensor* get(const std::string& name, int64_t numel) {
        for (int i = 0; i < n; ++i)
            if (t[i].name && name == t[i].name) {
                if (t[i].numel != numel) { ok = false; *err = "shape mismatch for " + name; return nullptr; }
                return &t[i];
            }
        ok = false; *err = "missing tensor " + name;
        return nullptr;
    }
};

// conv3x3 [cout][cin][3][3] (+ optional BN prefix) -> [cin][9][cout] with the BN scale folded in
uint16_t to_f16(float x) {          // IEEE fp32 -> fp16, round to nearest even, saturating to +-65504
    uint32_t u;
    memcpy(&u, &x, 4);
    const uint32_t sign = (u >> 16) & 0x8000u;
    u &= 0x7FFFFFFFu;
    if (u >= 0x477FF000u) return (uint16_t)(sign | 0x7BFFu);               // >= 65520 (or inf/nan): clamp
    if (u < 0x38800000u) {                                                 // subnormal half or zero
        if (u < 0x33000000u) return (uint16_t)sign;
        const int shift = 126 - (int)(u >> 23);                            // 14..24
        uint32_t mant = (u & 0x7FFFFFu) | 0x800000u;
        const uint32_t lsb = 1u << shift, half = lsb >> 1;
        uint32_t q = mant >> shift;
        const uint32_t rem = mant & (lsb - 1);
        if (rem > half || (rem == half && (q & 1))) ++q;
        return (uint16_t)(sign | q);
    }
    uint32_t e = ((u >> 23) - 112) << 10, m = (u >> 13) & 0x3FFu;
    uint32_t h = e | m;
    const uint32_t rem = u & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1))) ++h;                 // may carry into the exponent: still correct
    return (uint16_t)(sign | h);
}

float f16_to_float(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1Fu, m = h & 0x3FFu, u;
    if (e == 0) {
        if (m == 0) u = sign;
        else { int sh = 0; while (!(m & 0x400u)) { m <<= 1; ++sh; } m &= 0x3FFu; u = sign | ((uint32_t)(113 - sh) << 23) | (m << 13); }
    } else if (e == 31) u = sign | 0x7F800000u | (m << 13);
    else u = sign | ((e + 112) << 23) | (m << 13);
    float f;
    memcpy(&f, &u, 4);
    return f;
}

constexpr int kWideImage = 3;       // pack_conv's `tc` for the x3 image of the wide towers (conv_wide.cu)
constexpr int kWide256Image = 4;    // the same for the 256-channel towers, one image per 128-output-channel half (conv_wide256.cu)
// pack_conv's `tc` for the towers of a route: none on the CUDA cores
int weight_image(TowerRoute t) {
    return t == TowerRoute::Wide256 ? kWide256Image : is_wide(t) ? kWideImage : state_layout(t);
}

bool pack_conv(Loader& L, const std::string& conv, const std::string& bn, int cin, int cout, int stride,
               std::vector<float>& blob, std::vector<ConvLayer>& layers, int tc = 0, int H = 0, int W = 0) {
    const MzTensor* w = L.get(conv + ".weight", (int64_t)cout * cin * 9);
    if (!w) return false;
    std::vector<double> scale(cout, 1.0), shift(cout, 0.0);
    if (!bn.empty()) {
        const MzTensor* g = L.get(bn + ".weight", cout);
        const MzTensor* b = L.get(bn + ".bias", cout);
        const MzTensor* m = L.get(bn + ".running_mean", cout);
        const MzTensor* v = L.get(bn + ".running_var", cout);
        if (!g || !b || !m || !v) return false;
        for (int c = 0; c < cout; ++c) {
            scale[c] = (double)g->data[c] / sqrt((double)v->data[c] + 1e-5);
            shift[c] = (double)b->data[c] - (double)m->data[c] * scale[c];
        }
    }
    ConvLayer l;
    l.cin = cin; l.cout = cout; l.stride = stride;
    l.w_off = blob.size();
    blob.resize(blob.size() + (size_t)cin * 9 * cout);
    float* dst = blob.data() + l.w_off;
    for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci)
            for (int tap = 0; tap < 9; ++tap)
                dst[((size_t)ci * 9 + tap) * cout + co] = (float)((double)w->data[((size_t)co * cin + ci) * 9 + tap] * scale[co]);
    if (!bn.empty()) {
        l.b_off = (long)blob.size();
        for (int c = 0; c < cout; ++c) blob.push_back((float)shift[c]);
    } else {
        l.b_off = -1;
    }
    while (blob.size() % 4) blob.push_back(0.0f);           // keep every layer 16-byte aligned
    l.tc_off = l.tc_table_off = l.tc_scale_off = -1;
    if (tc == kLayoutSplit || tc == kWideImage || tc == kWide256Image) {
        // x3 image [tap][K-half][2C rows][cin 64]: rows 0..C-1 = w_h of cout 0..C-1, rows C..2C-1 = w_l; w' = w * 2^k with
        // k per output channel such that the row's largest |w'| lies in [1, 2); w_h = fp16(w'), w_l = fp16(w' - w_h).
        // The 16-byte chunks of a row are XOR-ed with row % 8 (wgmma K-major SWIZZLE_128B).  64 channels (conv_x3.cu): one
        // K-half; 128 (conv_wide.cu): two, each (tap, K-half) one 32 KB stage of the kernel's weight ring.  256
        // (conv_wide256.cu): per 128-output-channel half [tap][K-quarter][256 rows: w_h | w_l of the half's couts][cin 64],
        // each (half, tap, K-quarter) one 32 KB stage; the halves follow one another.
        const int C = cout;
        const bool wide = tc == kWideImage || tc == kWide256Image, halves = tc == kWide256Image;
        l.tc_off = (long)blob.size();
        blob.resize(blob.size() + (size_t)9 * 2 * C * C / 2);
        l.tc_scale_off = (long)blob.size();
        blob.resize(blob.size() + (size_t)C, 1.0f);
        uint16_t* img = reinterpret_cast<uint16_t*>(blob.data() + l.tc_off);
        float* undo = blob.data() + l.tc_scale_off;
        for (int co = 0; co < C; ++co) {
            float mx = 0.0f;
            for (int ci = 0; ci < C; ++ci)
                for (int tap = 0; tap < 9; ++tap)
                    mx = std::max(mx, fabsf((float)((double)w->data[((size_t)co * cin + ci) * 9 + tap] * scale[co])));
            int k = 0;
            if (mx > 0.0f && std::isfinite(mx)) { int e; frexpf(mx, &e); k = 1 - e; }      // mx * 2^k in [1, 2)
            if (k > 100) k = 100;
            if (k < -100) k = -100;
            undo[co] = ldexpf(1.0f, -k);
            for (int tap = 0; tap < 9; ++tap)
                for (int ci = 0; ci < C; ++ci) {
                    const float wf = (float)((double)w->data[((size_t)co * cin + ci) * 9 + tap] * scale[co]);   // the fp32 path's weight
                    const float ws = ldexpf(wf, k);
                    const uint16_t hb = to_f16(ws);
                    const float back = f16_to_float(hb);
                    const uint16_t lb = to_f16(ws - back);
                    const int cl = ci & 63;
                    const size_t col = (size_t)((((cl >> 3) ^ (co & 7))) << 3) + (cl & 7);
                    const size_t stage = (size_t)tap * (C / 64) + (ci >> 6);
                    if (halves) {
                        const size_t at = (((size_t)(co >> 7) * 9 * (C / 64) + stage) * 256 + (co & 127)) * 64 + col;
                        img[at] = hb;
                        img[at + 128 * 64] = lb;
                        continue;
                    }
                    img[(stage * 2 * C + co) * 64 + col] = hb;
                    img[(stage * 2 * C + C + co) * 64 + col] = lb;
                }
        }
        if (cin == C + 1) {
            // per board position (P64 row (y + 1) * 8 + x, or y * W + x on the wide towers' dense boards)
            l.tc_table_off = (long)blob.size();
            blob.resize(blob.size() + (size_t)(wide ? H * W : 64) * C, 0.0f);
            float* tab = blob.data() + l.tc_table_off;
            for (int y = 0; y < H; ++y)
                for (int x = 0; x < W; ++x)
                    for (int co = 0; co < C; ++co) {
                        double acc = 0.0;
                        for (int dy = -1; dy <= 1; ++dy)
                            for (int dx = -1; dx <= 1; ++dx)
                                if (y + dy >= 0 && y + dy < H && x + dx >= 0 && x + dx < W)
                                    acc += (double)w->data[((size_t)co * cin + C) * 9 + (dy + 1) * 3 + (dx + 1)] * scale[co];
                        tab[(size_t)(wide ? y * W + x : (y + 1) * 8 + x) * C + co] = (float)acc;
                    }
        }
    } else if (tc) {
        // fp16 image [tap][cout][cin] over the first 64 input channels, the 16-byte chunks of a cout row XOR-ed with
        // cout % 8 (wgmma K-major SWIZZLE_128B; two halves per float slot of the blob); an extra (65th) input channel
        // is the constant action plane and becomes a per-position fp32 table (sum of the taps that stay inside the board)
        const int C = cout;
        l.tc_off = (long)blob.size();
        blob.resize(blob.size() + (size_t)9 * C * C / 2);
        uint16_t* img = reinterpret_cast<uint16_t*>(blob.data() + l.tc_off);
        for (int tap = 0; tap < 9; ++tap)
            for (int ci = 0; ci < C; ++ci)
                for (int co = 0; co < C; ++co)
                    img[((size_t)tap * C + co) * C + ((((ci >> 3) ^ (co & 7))) << 3) + (ci & 7)] =
                        to_f16((float)((double)w->data[((size_t)co * cin + ci) * 9 + tap] * scale[co]));
        if (cin == C + 1) {
            l.tc_table_off = (long)blob.size();
            blob.resize(blob.size() + (size_t)64 * C, 0.0f);
            float* tab = blob.data() + l.tc_table_off;
            for (int y = 0; y < H; ++y)
                for (int x = 0; x < W; ++x)
                    for (int co = 0; co < C; ++co) {
                        double acc = 0.0;
                        for (int dy = -1; dy <= 1; ++dy)
                            for (int dx = -1; dx <= 1; ++dx)
                                if (y + dy >= 0 && y + dy < H && x + dx >= 0 && x + dx < W)
                                    acc += (double)w->data[((size_t)co * cin + C) * 9 + (dy + 1) * 3 + (dx + 1)] * scale[co];
                        tab[((y + 1) * 8 + x) * C + co] = (float)acc;
                    }
        }
    }
    layers.push_back(l);
    return true;
}

bool pack_resblock(Loader& L, const std::string& p, int ch, std::vector<float>& blob, std::vector<ConvLayer>& layers,
                   int tc = 0) {
    return pack_conv(L, p + ".conv1", p + ".bn1", ch, ch, 1, blob, layers, tc) &&
           pack_conv(L, p + ".conv2", p + ".bn2", ch, ch, 1, blob, layers, tc);
}

// DownSample's 18 convs under the prefix dp, in the order Runner::downsample runs them: conv1, resblocks1 x2, conv2,
// resblocks2 x3, resblocks3 x3.  Without `bn` (mz_debug_downsample) a block's conv takes the bias "<conv>.bias" instead
// of a BatchNorm.
bool pack_downsample(Loader& L, const std::string& dp, int obs_c, int C, bool bn, std::vector<float>& blob,
                     std::vector<ConvLayer>& layers) {
    auto conv = [&](const std::string& c, const std::string& norm, int ch) {
        if (bn) return pack_conv(L, c, norm, ch, ch, 1, blob, layers);
        const MzTensor* b = L.get(c + ".bias", ch);
        if (!b || !pack_conv(L, c, "", ch, ch, 1, blob, layers)) return false;
        layers.back().b_off = (long)blob.size();
        blob.insert(blob.end(), b->data, b->data + ch);                  // (ch % 4 == 0: stays aligned)
        return true;
    };
    auto block = [&](const std::string& p, int ch) { return conv(p + ".conv1", p + ".bn1", ch) && conv(p + ".conv2", p + ".bn2", ch); };
    bool ok = pack_conv(L, dp + ".conv1", "", obs_c, C / 2, 2, blob, layers);
    for (int i = 0; ok && i < 2; ++i) ok = block(dp + ".resblocks1." + std::to_string(i), C / 2);
    ok = ok && pack_conv(L, dp + ".conv2", "", C / 2, C, 2, blob, layers);
    for (int i = 0; ok && i < 3; ++i) ok = block(dp + ".resblocks2." + std::to_string(i), C);
    for (int i = 0; ok && i < 3; ++i) ok = block(dp + ".resblocks3." + std::to_string(i), C);
    return ok;
}

bool pack_head(Loader& L, const std::string& conv, const std::string& fc, int C, int rc, int HW, const int32_t* hidden,
               int n_hidden, int n_out, std::vector<float>& blob, HeadDesc& d) {
    const MzTensor* w = L.get(conv + ".weight", (int64_t)rc * C);
    const MzTensor* b = L.get(conv + ".bias", rc);
    if (!w || !b) return false;
    size_t size = blob.size();
    layout_head(C, rc, HW, hidden, n_hidden, n_out, &size, d);
    blob.resize(size, 0.0f);
    std::copy(w->data, w->data + (size_t)rc * C, blob.begin() + d.w1_off);
    std::copy(b->data, b->data + rc, blob.begin() + d.b1_off);
    for (int l = 0; l < d.mlp.n; ++l) {
        const int in = d.mlp.in[l], out = d.mlp.out[l];
        const MzTensor* lw = L.get(fc + "." + std::to_string(2 * l) + ".weight", (int64_t)in * out);
        const MzTensor* lb = L.get(fc + "." + std::to_string(2 * l) + ".bias", out);
        if (!lw || !lb) return false;
        float* dst = blob.data() + d.mlp.w_off[l];
        for (int o = 0; o < out; ++o)
            for (int i = 0; i < in; ++i) dst[((size_t)(i / 4) * out + o) * 4 + (i % 4)] = lw->data[(size_t)o * in + i];
        std::copy(lb->data, lb->data + out, blob.begin() + d.mlp.b_off[l]);
    }
    return true;
}
}  // namespace

int resnet_load_weights(ResNetDevice* r, const MzTensor* tensors, int n, std::string* err) {
    const MzNetDesc& nd = r->net;
    const int C = nd.channels, HW = r->hh * r->hw, F = 2 * nd.support_size + 1;
    Loader L{tensors, n, err};
    std::vector<float> conv, head;
    r->rep_down.clear(); r->rep_trunk.clear(); r->dyn.clear(); r->pred.clear();
    const std::string rp = "representation_network.module";
    bool ok = true;
    if (nd.downsample == 2) {
        // DownsampleCNN (models.py:278-297): features.0 = conv1, features.3 = conv2, both with bias and no BN
        const std::string fp = rp + ".downsample_net.features.";
        const int k = 2 * r->hh, mid = (nd.obs_c + C) / 2;
        const MzTensor* w1 = L.get(fp + "0.weight", (int64_t)mid * nd.obs_c * k * k);
        const MzTensor* b1 = L.get(fp + "0.bias", mid);
        const MzTensor* w2 = L.get(fp + "3.weight", (int64_t)C * mid * 25);
        const MzTensor* b2 = L.get(fp + "3.bias", C);
        ok = w1 && b1 && w2 && b2;
        if (ok) r->cnn = cnn_stem_pack(w1->data, b1->data, w2->data, b2->data, nd.obs_c, mid, C, k, conv);
    } else if (nd.downsample) {
        ok = pack_downsample(L, rp + ".downsample_net", nd.obs_c, C, true, conv, r->rep_down);
    } else {
        ok = ok && pack_conv(L, rp + ".conv", rp + ".bn", nd.obs_c, C, 1, conv, r->rep_trunk);
    }
    // the image of the route's tensor-core towers; the CUDA-core kernels read the fp32 weights, which every route packs,
    // so the range guard can switch to them without reloading
    const int tc = weight_image(r->route);
    for (int i = 0; ok && i < nd.blocks; ++i) ok = pack_resblock(L, rp + ".resblocks." + std::to_string(i), C, conv, r->rep_trunk, tc);
    const std::string dp = "dynamics_network.module";
    ok = ok && pack_conv(L, dp + ".conv", dp + ".bn", C + 1, C, 1, conv, r->dyn, tc, r->hh, r->hw);
    for (int i = 0; ok && i < nd.blocks; ++i) ok = pack_resblock(L, dp + ".resblocks." + std::to_string(i), C, conv, r->dyn, tc);
    const std::string pp = "prediction_network.module";
    for (int i = 0; ok && i < nd.blocks; ++i) ok = pack_resblock(L, pp + ".resblocks." + std::to_string(i), C, conv, r->pred, tc);
    ok = ok && pack_head(L, dp + ".conv1x1_reward", dp + ".fc", C, nd.reduced_reward, HW, nd.res_fc_reward, nd.n_res_fc_reward, F, head, r->reward_head);
    ok = ok && pack_head(L, pp + ".conv1x1_value", pp + ".fc_value", C, nd.reduced_value, HW, nd.res_fc_value, nd.n_res_fc_value, F, head, r->value_head);
    ok = ok && pack_head(L, pp + ".conv1x1_policy", pp + ".fc_policy", C, nd.reduced_policy, HW, nd.res_fc_policy, nd.n_res_fc_policy, nd.action_space, head, r->policy_head);
    if (!ok || !L.ok) return MZ_EINVAL;
    if (r->d_conv) cudaFree(r->d_conv);
    if (r->d_head) cudaFree(r->d_head);
    r->d_conv = r->d_head = nullptr;
    if (cudaMalloc(&r->d_conv, conv.size() * 4 + 64) != cudaSuccess || cudaMalloc(&r->d_head, head.size() * 4 + 64) != cudaSuccess) {
        *err = "weight allocation failed"; return MZ_ENOMEM;
    }
    cudaMemcpy(r->d_conv, conv.data(), conv.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(r->d_head, head.data(), head.size() * 4, cudaMemcpyHostToDevice);
    r->loaded = true;
    return MZ_OK;
}

// launch plan of one heads call (Runner::plan_heads); groups / threads / grid / smem are 0 on the generic route
struct HeadsPlan { int route = 0, groups = 0, threads = 0, grid = 0; size_t smem = 0; };

namespace {
// One tower call site of the network: the layers it runs, whether the first of them is a stem conv, and where its input
// lives.  Every tower family (tower_tc, small_tower, wide_tower, the per-layer convs of site_tower) takes it.
struct TowerSite {
    const std::vector<ConvLayer>* layers;
    size_t first;                  // first layer run; a stem (if any) and then 2 x blocks convs
    bool stem;
    int in_channels, H, W;         // the input board's planes (the dynamics stem adds the action plane)
    const float* in;               // scratch, or in search the hidden-state pool, which stays read only
    const int32_t* gather_parent;  // in search: game g reads slot gather_parent[g] of pool_stride
    int pool_stride;
    const int32_t* action;         // the dynamics stem's action plane
};

struct Runner {
    ResNetDevice* r; cudaStream_t stream; int64_t* launches; std::string* err; int n;
    int g0 = 0;                // games [g0, g0 + n) of the batch (partitioned replay); buffers are addressed by the global index
    SmallTowerPlan* small_plan = nullptr;   // when set, small_tower reports the plan of its launch here (mz_debug_small_tower)
    int heads_route = MZ_HEADS_PLANNED;     // mz_debug_heads only: force a heads route; the network never sets it
    HeadsPlan* heads_plan_out = nullptr;    // when set, heads reports the plan of its launch here (mz_debug_heads)
    WideTowerPlan* wide_plan_out = nullptr; // when set, wide_tower reports the plan of its launch here (mz_debug_wide_tower)
    Wide256Plan* wide256_plan_out = nullptr; // the same for the 256-channel towers (mz_debug_wide256_tower)
    int wide256_boards = 0;                 // mz_debug_wide256_tower only: force the boards per CTA pair; 0 = planned
    bool fail(const char* what, cudaError_t e) { *err = std::string(what) + ": " + cudaGetErrorString(e); return false; }

    // conv: in -> out. `in` may be gathered from the pool; action adds the constant plane.
    TowerLayer tower_layer(const ConvLayer& l, int in_buf, int out_buf, int res_buf, bool relu) {
        TowerLayer t{};
        t.w = r->d_conv + l.tc_off;
        t.bias = l.b_off >= 0 ? r->d_conv + l.b_off : nullptr;
        t.action_table = l.tc_table_off >= 0 ? r->d_conv + l.tc_table_off : nullptr;
        t.scale = l.tc_scale_off >= 0 ? r->d_conv + l.tc_scale_off : nullptr;
        t.in_buf = in_buf; t.out_buf = out_buf; t.res_buf = res_buf; t.relu = relu ? 1 : 0;
        return t;
    }

    bool launch_tower(TowerArgs& a) {
        a.n = n; a.H = r->hh; a.W = r->hw; a.A = r->net.action_space;
        static const int dbg = getenv("MZ_TC_DEBUG_SKIP") ? atoi(getenv("MZ_TC_DEBUG_SKIP")) : 0;
        a.debug_skip = dbg;
        a.g0 = g0; a.sat_count = r->d_sat;
        const bool x3 = r->route == TowerRoute::TcX3;
        kt_begin(KT_TOWER, stream);
        cudaError_t e = x3 ? launch_conv_tower_x3(a, r->sm_count, stream) : launch_conv_tower_tc(a, r->sm_count, stream);
        kt_end(stream);
        if (e != cudaSuccess) return fail("conv_tower_tc launch", e);
        *launches += x3 ? conv_x3_launches(n, r->sm_count) : 1;
        return true;
    }

    // one tensor-core conv (a tower of one layer)
    bool conv_tc(const ConvLayer& l, const float* in, float* out, const float* residual, bool relu,
                 const int32_t* gather_parent = nullptr, int pool_stride = 0, const int32_t* action = nullptr) {
        TowerArgs a{};
        a.n_layers = 1;
        a.buf[0] = const_cast<float*>(in); a.buf[1] = out; a.buf[2] = const_cast<float*>(residual);
        a.layer[0] = tower_layer(l, 0, 1, residual ? 2 : -1, relu);
        if (!action) a.layer[0].action_table = nullptr;
        a.gather_parent = gather_parent; a.pool_stride = pool_stride; a.action = action;
        return launch_tower(a);
    }

    bool blocks_tc(const std::vector<ConvLayer>& layers, size_t first, size_t count, float** cur, float** tmp, float** spare) {
        for (size_t b = 0; b < count; ++b) {
            if (!conv_tc(layers[first + 2 * b], *cur, *tmp, nullptr, true)) return false;
            if (!conv_tc(layers[first + 2 * b + 1], *tmp, *spare, *cur, true)) return false;
            float* t = *cur; *cur = *spare; *spare = t;
        }
        return true;
    }

    // The tower of a site in as few persistent launches as possible, its input s.in (in the board layout) followed by
    // the three workspaces.  Returns the buffer holding the result (one of the workspaces, or s.in if there was nothing
    // to do) or nullptr on error.
    const float* tower_tc(const TowerSite& s) {
        const std::vector<ConvLayer>& layers = *s.layers;
        float* const* ws = r->ws;
        const float* ext = s.in;
        const int32_t *gather_parent = s.gather_parent, *action = s.action;
        const int pool_stride = s.pool_stride;
        const bool stem = s.stem;
        size_t count = r->net.blocks;
        if (r->route != TowerRoute::TcX3 && n > conv_tc_max_boards_fused(r->sm_count)) {
            // too many tiles per CTA for the fused mode: one launch per conv
            float* free_ws[3]; int nf = 0;
            for (int i = 0; i < 3; ++i) if (ws[i] != ext) free_ws[nf++] = ws[i];
            if (nf < 3) free_ws[nf++] = const_cast<float*>(ext);      // ext is itself a workspace: reusable as the third
            float *cur = free_ws[0], *tmp = free_ws[1], *spare = free_ws[2];
            size_t first = s.first;
            // (the result buffer may be ext itself when ext is one of the workspaces: whether any layer ran decides
            // what is returned, not a comparison with ext)
            const bool any = stem || count > 0;
            if (stem) { if (!conv_tc(layers[first], ext, cur, nullptr, true, gather_parent, pool_stride, action)) return nullptr; first += 1; }
            if (count > 0 && !stem) {
                if (!conv_tc(layers[first], ext, tmp, nullptr, true, gather_parent, pool_stride)) return nullptr;
                if (!conv_tc(layers[first + 1], tmp, spare, ext, true)) return nullptr;      // residual = ext (plain addressing only)
                { float* t = cur; cur = spare; spare = t; }
                first += 2; count -= 1;
            }
            if (!blocks_tc(layers, first, count, &cur, &tmp, &spare)) return nullptr;
            return any ? cur : ext;
        }
        size_t li = s.first, blocks_left = count;
        bool stem_left = stem;
        const float* ext_now = ext;                 // buf[0] of the next launch
        const int32_t* gather_now = gather_parent;
        const float* result = ext;
        while (stem_left || blocks_left > 0) {
            TowerArgs a{};
            a.buf[0] = const_cast<float*>(ext_now);
            // the three workspaces, skipping the one that currently holds the input
            int nb = 1;
            for (int i = 0; i < 3; ++i) if (ws[i] != ext_now) a.buf[nb++] = ws[i];
            if (nb < 4) a.buf[nb++] = nullptr;      // (only two spare workspaces when the input is one of ws)
            a.gather_parent = gather_now; a.pool_stride = pool_stride; a.action = action;
            int cur = 0, nl = 0;
            // the input buffer is dead after its last reader: always so for a workspace written by the previous launch and
            // for the tower's own scratch input, never for a gathered pool
            const bool reuse0 = !gather_now;
            auto pick = [&](int avoid1, int avoid2) {
                for (int i = 1; i < 4; ++i) if (i != avoid1 && i != avoid2 && a.buf[i]) return i;
                if (reuse0 && avoid1 != 0 && avoid2 != 0) return 0;
                return -1;
            };
            if (stem_left) {
                const int o = pick(cur, -1);
                a.layer[nl++] = tower_layer(layers[li++], cur, o, -1, true);
                cur = o; stem_left = false;
            }
            while (blocks_left > 0 && nl + 2 <= kTowerMaxLayers) {
                const int t1 = pick(cur, -1);
                const int t2 = pick(cur, t1);
                if (t1 < 0 || t2 < 0) break;
                a.layer[nl++] = tower_layer(layers[li++], cur, t1, -1, true);
                a.layer[nl++] = tower_layer(layers[li++], t1, t2, cur, true);
                cur = t2; --blocks_left;
            }
            if (nl == 0) { *err = "tower_tc: no workspace left"; return nullptr; }
            for (int i = 0; i < nl; ++i) if (!action) a.layer[i].action_table = nullptr;
            a.n_layers = nl;
            if (!launch_tower(a)) return nullptr;
            result = a.buf[cur];
            ext_now = result; gather_now = nullptr;
        }
        return result;
    }

    // The four tower call sites of the network (the debug towers run the same descriptions).  Representation: from the
    // observation planes through the stem or, after_stem, from the stem's output (the tensor-core and wide towers leave
    // the stem to conv3x3_kernel); the trunk of a downsampled net is blocks only, on the DownSample output.
    TowerSite representation_site(const float* in, bool after_stem = false) const {
        if (!r->net.downsample && !after_stem)
            return TowerSite{&r->rep_trunk, 0, true, r->net.obs_c, r->net.obs_h, r->net.obs_w, in, nullptr, 0, nullptr};
        return TowerSite{&r->rep_trunk, after_stem ? 1u : 0u, false, r->C, r->hh, r->hw, in, nullptr, 0, nullptr};
    }
    // Dynamics: the stem reads the states and the action plane; in search game g's state is slot gather_parent[g] of
    // the pool `in`.
    TowerSite dynamics_site(const float* in, const int32_t* action, const int32_t* gather_parent = nullptr,
                            int pool_stride = 0) const {
        return TowerSite{&r->dyn, 0, true, r->C, r->hh, r->hw, in, gather_parent, pool_stride, action};
    }
    // Prediction: blocks only, on the rescaled state.
    TowerSite prediction_site(const float* in) const {
        return TowerSite{&r->pred, 0, false, r->C, r->hh, r->hw, in, nullptr, 0, nullptr};
    }

    bool conv(const ConvLayer& l, const float* in, float* out, const float* residual, bool relu, int Hin, int Win,
              const int32_t* gather_parent = nullptr, int pool_stride = 0, const int32_t* action = nullptr,
              bool out_p64c4 = false) {
        if (g0 != 0) { *err = "conv3x3: partitioned calls are not supported on the per-layer route"; return false; }
        ConvArgs a{};
        a.out_p64c4 = out_p64c4 ? state_layout(r->route) : 0;
        a.in = in; a.out = out; a.residual = residual; a.w = r->d_conv + l.w_off;
        a.bias = l.b_off >= 0 ? r->d_conv + l.b_off : nullptr;
        a.gather_parent = gather_parent; a.pool_stride = pool_stride; a.action = action;
        a.n = n; a.Cin = l.cin; a.Cout = l.cout; a.Hin = Hin; a.Win = Win; a.stride = l.stride;
        a.Ho = conv_out(Hin, l.stride); a.Wo = conv_out(Win, l.stride); a.relu = relu; a.A = r->net.action_space;
        ConvPlan plan;
        if (!conv3x3_plan(n, l.cin, l.cout, Hin, Win, l.stride, &plan, err)) return false;
        const int P = plan.P, threads = kConvThreads;
        a.band_rows = plan.band_rows; a.boards_per_cta = plan.boards; a.cin_chunk = plan.cin_chunk; a.cout_tile = plan.cout_tile;
        const size_t smem = plan.smem;
        const dim3 grid = plan.grid;
        const bool multi = plan.max_items == 4;
#define MZ_CONV(PP, SS)                                                                                         \
        if (P == PP && l.stride == SS) {                                                                        \
            auto kern = multi ? conv3x3_kernel<PP, SS, 4> : conv3x3_kernel<PP, SS, 1>;                          \
            static size_t attr_smem[2] = {0, 0};                                                                \
            if (attr_smem[multi] < smem) {                                                                      \
                cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
                if (e != cudaSuccess) return fail("conv attr", e);                                              \
                attr_smem[multi] = smem;                                                                        \
            }                                                                                                   \
            kt_begin(KT_CONV, stream);                                                                          \
            kern<<<grid, threads, smem, stream>>>(a);                                                           \
            kt_end(stream);                                                                                     \
        }
        MZ_CONV(8, 1) MZ_CONV(7, 1) MZ_CONV(6, 1) MZ_CONV(4, 1) MZ_CONV(3, 1) MZ_CONV(2, 1) MZ_CONV(1, 1)
        MZ_CONV(8, 2) MZ_CONV(6, 2) MZ_CONV(4, 2) MZ_CONV(3, 2) MZ_CONV(2, 2) MZ_CONV(1, 2) MZ_CONV(7, 2)
#undef MZ_CONV
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail("conv3x3 launch", e);
        *launches += 1;
        return true;
    }

    // DownsampleCNN stem of the observations `in`: stage 1 into `pooled`, stage 2 into `out` (cnn_stem.cu)
    bool cnn_stem(const float* in, float* pooled, float* out) {
        CnnStemPlan p;
        if (!cnn_stem_plan(n, r->net.obs_c, r->C, r->net.obs_h, r->net.obs_w, r->sm_count, &p, err)) return false;
        kt_begin(KT_CONV, stream);
        cudaError_t e = cnn_stem_launch(p, r->d_conv, r->cnn, in, pooled, out, n, stream);
        kt_end(stream);
        if (e != cudaSuccess) return fail("cnn stem launch", e);
        *launches += 2;
        return true;
    }

    // arguments of the fused CUDA-core tower of a site writing `out`; false when the layers are not of the supported kind
    bool small_tower_args(SmallTowerArgs& a, const TowerSite& s, float* out) {
        const size_t nl = (s.stem ? 1 : 0) + 2 * (size_t)r->net.blocks;
        if (nl == 0 || nl > (size_t)kSmallTowerMaxLayers) return false;
        a = SmallTowerArgs{};
        a.in = s.in; a.out = out; a.blob = r->d_conv; a.gather_parent = s.gather_parent; a.action = s.action;
        a.pool_stride = s.pool_stride;
        a.n = n; a.g0 = g0; a.C = r->C; a.H = s.H; a.W = s.W; a.A = r->net.action_space; a.in_channels = s.in_channels;
        a.n_layers = (int)nl;
        for (size_t i = 0; i < nl; ++i) {
            const ConvLayer& l = (*s.layers)[s.first + i];
            if (l.stride != 1 || l.cout != r->C) return false;
            SmallTowerLayer& t = a.layer[i];
            t.w_off = (int)l.w_off; t.b_off = (int)l.b_off; t.cin = l.cin; t.relu = 1;
            t.residual = (i >= (s.stem ? 1u : 0u) && ((i - (s.stem ? 1 : 0)) & 1)) ? 1 : 0;     // second conv of a block
        }
        return true;
    }

    // The tower of a site as ONE fused CUDA-core launch (small_tower.cu).  Returns 1 = launched, 0 = shape not supported
    // (the caller falls back to one launch per conv), -1 = error.
    int small_tower(const TowerSite& s, float* out, bool dry_run = false) {
        if (!r->fuse_small) return 0;
        SmallTowerArgs a{};
        if (!small_tower_args(a, s, out)) return 0;
        if (!small_tower_supported(a)) return 0;
        if (dry_run) return 1;
        kt_begin(KT_SMALL, stream);
        cudaError_t e = launch_small_tower(a, r->sm_count, stream, small_plan);
        kt_end(stream);
        if (e != cudaSuccess) { fail("small_tower launch", e); return -1; }
        *launches += 1;
        return 1;
    }

    // the arguments every wide tower launch shares (WideTowerArgs, Wide256Args) of a site with nl layers writing `out`
    template <typename Args>
    void wide_args(Args& a, const TowerSite& s, float* out, int nl) {
        a.in = s.in; a.out = out; a.gather_parent = s.gather_parent; a.pool_stride = s.pool_stride; a.action = s.action;
        a.n = n; a.H = r->hh; a.W = r->hw; a.A = r->net.action_space; a.g0 = g0; a.stem = s.stem ? 1 : 0; a.n_layers = nl;
        a.sat_count = r->d_sat;
        for (int i = 0; i < nl; ++i) {
            const ConvLayer& l = (*s.layers)[s.first + i];
            WideLayer& t = a.layer[i];
            t.w = r->d_conv + l.tc_off;
            t.scale = r->d_conv + l.tc_scale_off;
            t.bias = l.b_off >= 0 ? r->d_conv + l.b_off : nullptr;
            t.action_table = i == 0 && s.stem && s.action && l.tc_table_off >= 0 ? r->d_conv + l.tc_table_off : nullptr;
        }
    }

    // The tower of a site of a 128-channel net as ONE x3 tensor-core launch (conv_wide.cu), dense NCHW in and out, one CTA
    // or (WidePair) one CTA pair per board; of a 256-channel net (Wide256, conv_wide256.cu) one CTA pair per group of
    // boards, each CTA computing half the output channels.  Returns what small_tower returns: 1 = launched, 0 = not the
    // wide route, -1 = error.
    int wide_tower(const TowerSite& s, float* out) {
        const int nl = (s.stem ? 1 : 0) + 2 * r->net.blocks;
        if (!is_wide(r->route) || nl == 0) return 0;
        const char* why = "";
        if (r->route == TowerRoute::Wide256) {
            Wide256Plan p;
            if (!wide256_plan(n, r->C, r->hh, r->hw, nl, r->sm_count, wide256_boards, &p, &why)) return 0;
            Wide256Args a{};
            wide_args(a, s, out, nl);
            if (wide256_plan_out) *wide256_plan_out = p;
            kt_begin(KT_TOWER, stream);
            cudaError_t e = launch_wide256_tower(a, p, stream);
            kt_end(stream);
            if (e != cudaSuccess) { fail("wide256 tower launch", e); return -1; }
            *launches += p.launches;
            return 1;
        }
        const bool pair = r->route == TowerRoute::WidePair;
        WideTowerPlan p;
        if (!(pair ? wide_pair_plan : wide_tower_plan)(n, r->C, r->hh, r->hw, nl, r->sm_count, &p, &why)) return 0;
        WideTowerArgs a{};
        wide_args(a, s, out, nl);
        if (wide_plan_out) *wide_plan_out = p;
        kt_begin(KT_TOWER, stream);
        cudaError_t e = pair ? launch_wide_pair_tower(a, p, stream) : launch_wide_tower(a, p, stream);
        kt_end(stream);
        if (e != cudaSuccess) { fail("wide tower launch", e); return -1; }
        *launches += p.launches;
        return 1;
    }

    // The tower of a site in resnet_inference: the wide launch and then the fused CUDA-core launch, as far as `tries`
    // names them, else one conv3x3_kernel per conv.  The workspaces *cur, *tmp, *spare rotate: a site with a stem writes
    // *cur first; one without reads s.in (*cur itself, or the rescaled state, which is never written) and writes *tmp
    // first.  Returns the buffer holding the result (s.in when the site has no layer), nullptr on error.
    enum { kTryWide = 1, kTryFused = 2 };
    const float* site_tower(const TowerSite& s, int tries, float** cur, float** tmp, float** spare) {
        float* out = s.stem ? *cur : *tmp;
        int done = (tries & kTryWide) ? wide_tower(s, out) : 0;
        if (done == 0 && (tries & kTryFused)) done = small_tower(s, out);
        if (done < 0) return nullptr;
        if (done) {
            if (out == *tmp) std::swap(*cur, *tmp);
            return *cur;
        }
        size_t li = s.first;
        const float* x = s.in;
        if (s.stem) {
            if (!conv((*s.layers)[li++], s.in, *cur, nullptr, true, s.H, s.W, s.gather_parent, s.pool_stride, s.action)) return nullptr;
            x = *cur;
        }
        for (int b = 0; b < r->net.blocks; ++b, li += 2) {
            if (!conv((*s.layers)[li], x, *tmp, nullptr, true, r->hh, r->hw)) return nullptr;
            if (!conv((*s.layers)[li + 1], *tmp, *spare, x, true, r->hh, r->hw)) return nullptr;
            std::swap(*cur, *spare);
            x = *cur;
        }
        return x;
    }

    // residual tower: layers[2k], layers[2k+1] are one block; x ends up in `*cur`
    bool blocks(const std::vector<ConvLayer>& layers, size_t first, size_t count, float** cur, float** tmp, float** spare, int H, int W) {
        for (size_t b = 0; b < count; ++b) {
            if (!conv(layers[first + 2 * b], *cur, *tmp, nullptr, true, H, W)) return false;
            if (!conv(layers[first + 2 * b + 1], *tmp, *spare, *cur, true, H, W)) return false;
            float* t = *cur; *cur = *spare; *spare = t;
        }
        return true;
    }

    // DownSample (models.py:233-275) of the observations `in`, r->rep_down's 24 convs and two pools: conv1 at stride 2
    // (no ReLU), resblocks1 x2 at C/2 channels, conv2 at stride 2, resblocks2 x3, pool, resblocks3 x3, pool.  The
    // workspaces rotate; the result is left in *cur.  With ds_stages set (mz_debug_downsample), the outputs of conv1,
    // resblocks1, conv2, resblocks2, the first pool and resblocks3 are copied there.
    float* const* ds_stages = nullptr;
    bool downsample(const float* in, float** cur, float** tmp, float** spare) {
        const std::vector<ConvLayer>& d = r->rep_down;
        const int C = r->C;
        int H = r->net.obs_h, W = r->net.obs_w, stage = 0;
        auto keep = [&](int channels) {
            if (!ds_stages) return true;
            cudaError_t e = cudaMemcpyAsync(ds_stages[stage++], *cur, (size_t)n * channels * H * W * 4, cudaMemcpyDeviceToDevice, stream);
            return e == cudaSuccess || fail("downsample stage copy", e);
        };
        if (!conv(d[0], in, *cur, nullptr, false, H, W)) return false;
        H = conv_out(H, 2); W = conv_out(W, 2);
        if (!keep(C / 2) || !blocks(d, 1, 2, cur, tmp, spare, H, W) || !keep(C / 2)) return false;
        if (!conv(d[5], *cur, *tmp, nullptr, false, H, W)) return false;
        std::swap(*cur, *tmp);
        H = conv_out(H, 2); W = conv_out(W, 2);
        if (!keep(C) || !blocks(d, 6, 3, cur, tmp, spare, H, W) || !keep(C)) return false;
        for (int pool = 0; pool < 2; ++pool) {
            const int Ho = conv_out(H, 2), Wo = conv_out(W, 2);
            const size_t total = (size_t)n * C * Ho * Wo;
            avgpool3x3s2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(*cur, *tmp, n * C, H, W, Ho, Wo);
            cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return fail("avgpool3x3s2 launch", e);
            *launches += 1;
            std::swap(*cur, *tmp);
            H = Ho; W = Wo;
            if (pool == 0 && (!keep(C) || !blocks(d, 12, 3, cur, tmp, spare, H, W) || !keep(C))) return false;
        }
        return true;
    }

    // heads whose weights do not fit in shared memory: one plain kernel per stage (see big_*_kernel above)
    bool heads_big(const float* x, int n_heads, const HeadDesc* const* hs, float* l0, float* l1, float* s0, float* s1,
                   float* rescaled, float* pool_hidden, int pool_stride, int out_slot) {
        const int C = r->C, HW = r->hh * r->hw, S = r->net.support_size;
        if (g0 != 0) { *err = "heads (generic route): partitioned calls are not supported"; return false; }
        kt_begin(KT_HEADS, stream);
        if (rescaled || pool_hidden) {
            big_rescale_kernel<<<(n * C + 127) / 128, 128, 0, stream>>>(x, n, C, HW, rescaled, pool_hidden, pool_stride, out_slot);
            *launches += 1;
        }
        float* logits_out[2] = {l0, l1};
        float* scalar_out[2] = {s0, s1};
        for (int hi = 0; hi < n_heads; ++hi) {
            const HeadDesc& d = *hs[hi];
            int width = ((d.rc * HW + 3) & ~3);
            for (int l = 0; l < d.mlp.n; ++l) width = std::max(width, (d.mlp.out[l] + 3) & ~3);
            const size_t need = (size_t)2 * n * width;
            if (r->big_elems < need) {
                if (r->big_scratch) cudaFree(r->big_scratch);
                r->big_scratch = nullptr; r->big_elems = 0;
                if (cudaMalloc(&r->big_scratch, need * 4 + 64) != cudaSuccess) { *err = "heads: scratch allocation failed"; kt_end(stream); return false; }
                r->big_elems = need;
            }
            float* cur = r->big_scratch;
            float* nxt = r->big_scratch + (size_t)n * width;
            cudaMemsetAsync(cur, 0, (size_t)n * width * 4, stream);           // zero padding behind rc*HW
            const size_t items = (size_t)n * d.rc * HW;
            big_conv1x1_kernel<<<(unsigned)((items + 127) / 128), 128, 0, stream>>>(x, r->d_head + d.w1_off, r->d_head + d.b1_off, n, C, d.rc, HW, cur, width);
            *launches += 1;
            for (int l = 0; l < d.mlp.n; ++l) {
                const int out4 = (d.mlp.out[l] + 3) & ~3;
                big_fc_kernel<<<(unsigned)(((size_t)n * out4 + 127) / 128), 128, 0, stream>>>(
                    cur, r->d_head + d.mlp.w_off[l], r->d_head + d.mlp.b_off[l], n, d.mlp.in[l], d.mlp.out[l], width, width,
                    l == d.mlp.n - 1 ? 0 : 1, nxt);
                *launches += 1;
                float* t = cur; cur = nxt; nxt = t;
            }
            big_scalar_kernel<<<(n * 32 + 127) / 128, 128, 0, stream>>>(cur, n, width, d.n_out, S, logits_out[hi], scalar_out[hi]);
            *launches += 1;
        }
        kt_end(stream);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail("heads (generic route)", e);
        return true;
    }

    // arguments of one heads launch (everything but the launch geometry); x and the states are in the route's layout
    HeadsArgs heads_args(const float* x, int n_heads, const HeadDesc* h0, const HeadDesc* h1, float* l0, float* l1, float* s0, float* s1,
                         float* rescaled, float* pool_hidden, int pool_stride, int out_slot, float* state_p64c4 = nullptr) {
        HeadsArgs a{};
        a.p64c4 = state_layout(r->route); a.W = r->hw; a.state_p64c4 = state_p64c4;
        a.x = x; a.blob = r->d_head; a.n = n; a.g0 = g0; a.C = r->C; a.HW = r->hh * r->hw; a.S = r->net.support_size;
        a.hw_inv = a.HW >= 2 ? (unsigned)((0x100000000ull + (unsigned)a.HW - 1u) / (unsigned)a.HW) : 0u;
        a.n_heads = n_heads;
        const HeadDesc* hs[2] = {h0, h1};
        for (int i = 0; i < n_heads; ++i) a.head[i] = *hs[i];
        a.logits[0] = l0; a.logits[1] = l1; a.scalar[0] = s0; a.scalar[1] = s1;
        a.rescaled = rescaled; a.pool_hidden = pool_hidden; a.pool_stride = pool_stride; a.out_slot = out_slot;
        const HeadsFootprint f = heads_footprint(a.C, a.HW, n_heads, hs);
        a.w_lo = f.w_lo; a.w_floats = f.w_floats; a.smem_floats = f.smem_floats; a.warp_floats = f.warp_floats;
        return a;
    }

    // Launch plan of one heads call (host only; the launch and mz_debug_heads_plan both take it from here).  One warp per
    // sample when a sample is small, 128 threads per sample otherwise; only as many groups per CTA as it takes to give
    // every SM work (1024 Connect4 boards: 147 CTAs x 7 groups, not 128 x 8), fewer while the weights and the groups' tiles
    // exceed shared memory; the generic route (dense layout, one range) when even one group does not fit.  heads_route
    // forces a route; false with the reason in *err when the forced route cannot take the call.
    bool plan_heads(const HeadsArgs& a, HeadsPlan* p) const {
        *p = HeadsPlan{};
        if (heads_route == MZ_HEADS_GENERIC) {
            if (a.p64c4) { *err = "heads: the generic route reads dense states only, not the tensor-core board layout"; return false; }
            if (a.g0 != 0) { *err = "heads (generic route): partitioned calls are not supported"; return false; }
            p->route = MZ_HEADS_GENERIC;
            return true;
        }
        const bool narrow = heads_route == MZ_HEADS_PLANNED ? a.C * a.HW <= 1024 && a.n_heads <= 2 : heads_route == MZ_HEADS_WARP;
        const int group = narrow ? 32 : 128;
        int groups = kHeadThreads / group;
        groups = std::max(1, std::min(groups, (n + r->sm_count - 1) / r->sm_count));
        size_t smem = ((size_t)a.w_floats + (size_t)groups * a.warp_floats) * 4;
        while (groups > 1 && smem > 227 * 1024) { --groups; smem = ((size_t)a.w_floats + (size_t)groups * a.warp_floats) * 4; }
        if (smem > 227 * 1024) {
            if (heads_route != MZ_HEADS_PLANNED) { *err = "heads: the forced group's weights + tile exceed shared memory"; return false; }
            if (a.p64c4) { *err = "heads: weights + tiles exceed shared memory"; return false; }
            if (a.g0 != 0) { *err = "heads (generic route): partitioned calls are not supported"; return false; }
            p->route = MZ_HEADS_GENERIC;
            return true;
        }
        p->route = narrow ? MZ_HEADS_WARP : MZ_HEADS_WIDE;
        p->groups = groups; p->threads = groups * group; p->smem = smem;
        p->grid = std::min((n + groups - 1) / groups, r->sm_count);
        return true;
    }

    bool heads(const float* x, int n_heads, const HeadDesc* h0, const HeadDesc* h1, float* l0, float* l1, float* s0, float* s1,
               float* rescaled, float* pool_hidden, int pool_stride, int out_slot, float* state_p64c4 = nullptr) {
        HeadsArgs a = heads_args(x, n_heads, h0, h1, l0, l1, s0, s1, rescaled, pool_hidden, pool_stride, out_slot, state_p64c4);
        const HeadDesc* hs[2] = {h0, h1};
        HeadsPlan plan;
        if (!plan_heads(a, &plan)) return false;
        if (heads_plan_out) *heads_plan_out = plan;
        if (plan.route == MZ_HEADS_GENERIC) return heads_big(x, n_heads, hs, l0, l1, s0, s1, rescaled, pool_hidden, pool_stride, out_slot);
        const bool narrow = plan.route == MZ_HEADS_WARP;
        const size_t smem = plan.smem;
        const int threads = plan.threads, grid = plan.grid;
        static size_t attr_smem[2] = {0, 0};
        if (attr_smem[narrow] < smem) {
            cudaError_t e0 = narrow ? cudaFuncSetAttribute(heads_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                                    : cudaFuncSetAttribute(heads_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e0 != cudaSuccess) return fail("heads attr", e0);
            attr_smem[narrow] = smem;
        }
        kt_begin(KT_HEADS, stream);
        cudaError_t e = narrow ? launch_chained(heads_kernel<32>, dim3(grid), dim3(threads), smem, stream, a)
                               : launch_chained(heads_kernel<128>, dim3(grid), dim3(threads), smem, stream, a);
        kt_end(stream);
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) return fail("heads launch", e);
        *launches += 1;
        return true;
    }

    // The three heads calls of resnet_inference / resnet_inference_tc (mz_debug_heads runs the same helpers).  On the
    // tensor-core route the input and the pool are in the board layout and the rescaled state is also written into
    // scratch_state, the prediction tower's input.  Representation: rescale only (no heads on the root state).
    bool representation_heads(const float* x, float* hidden, float* pool_hidden, int pool_stride, int out_slot) {
        return heads(x, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, hidden, pool_hidden, pool_stride, out_slot,
                     tc_state());
    }
    // Dynamics (plain API call and in search): reward head on the raw state + rescale.
    bool dynamics_heads(const float* x, float* reward_logits, float* reward, float* hidden, float* pool_hidden, int pool_stride,
                        int out_slot) {
        return heads(x, 1, &r->reward_head, nullptr, reward_logits, nullptr, reward, nullptr, hidden, pool_hidden, pool_stride,
                     out_slot, tc_state());
    }
    // Prediction: value and policy heads on the prediction tower's output (a scalar for the value only).
    bool prediction_heads(const float* x, float* value_logits, float* policy_logits, float* value) {
        return heads(x, 2, &r->value_head, &r->policy_head, value_logits, policy_logits, value, nullptr, nullptr, nullptr, 0, 0);
    }
    float* tc_state() const { return is_tc(r->route) ? r->scratch_state : nullptr; }
};
}  // namespace

// Where resnet_inference_tc leaves the input of a tensor-core tower: the representation stem's output, the converted
// dense states of a plain dynamics call, the rescaled state the heads wrote (in search the dynamics tower reads the pool)
static float* tc_tower_input(ResNetDevice* r, int site) {
    return site == MZ_TOWER_REPRESENTATION ? r->ws[0] : site == MZ_TOWER_DYNAMICS ? r->ws[2] : r->scratch_state;
}

// Tensor-core variant: every C->C conv of the three towers runs in conv_tc.cu on the P64C4 layout; the
// stem conv (obs -> C) and the heads stay on the CUDA-core kernels above, reading / writing that layout.
static int resnet_inference_tc(ResNetDevice* r, const InferCall& c, cudaStream_t stream, int64_t* launches, std::string* err) {
    const MzNetDesc& nd = r->net;
    const int n = c.n, C = r->C, hh = r->hh, hw = r->hw, F = 2 * nd.support_size + 1;
    Runner R{r, stream, launches, err, n, c.g0};
    if (c.g0 != 0 && (r->route != TowerRoute::TcX3 || !c.recurrent || !c.gather_parent)) { *err = "resnet: partitioned calls need the x3 towers in pool mode"; return MZ_EINVAL; }
    float* state = r->scratch_state;                   // rescaled state, P64C4, input of the prediction tower
    if (!c.recurrent) {
        float* stem_out = tc_tower_input(r, MZ_TOWER_REPRESENTATION);
        if (!R.conv(r->rep_trunk[0], c.in, stem_out, nullptr, true, nd.obs_h, nd.obs_w, nullptr, 0, nullptr, true)) return MZ_ECUDA;
        const float* x = R.tower_tc(R.representation_site(stem_out, true));
        if (!x) return MZ_ECUDA;
        if (!R.representation_heads(x, c.hidden, c.pool_hidden, c.pool_stride, c.out_slot)) return MZ_ECUDA;
        if (c.reward_logits) {
            fill_root_reward_logits_kernel<<<(n * F + 255) / 256, 256, 0, stream>>>(c.reward_logits, n, F, nd.support_size);
            *launches += 1;
        }
        if (c.reward) {
            fill_root_reward_kernel<<<(n + 255) / 256, 256, 0, stream>>>(c.reward, n);
            *launches += 1;
        }
    } else {
        const float* x;
        if (c.gather_parent) {
            x = R.tower_tc(R.dynamics_site(c.pool_hidden, c.action, c.gather_parent, c.pool_stride));
        } else {
            // plain API call: dense NCHW hidden states -> P64C4
            const size_t total = (size_t)n * C * hh * hw;
            float* staged = tc_tower_input(r, MZ_TOWER_DYNAMICS);
            nchw_to_p64c4_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(c.in, staged, n, C, hh, hw,
                                                                                       r->route == TowerRoute::TcX3);
            *launches += 1;
            x = R.tower_tc(R.dynamics_site(staged, c.action));
        }
        if (!x) return MZ_ECUDA;
        if (!R.dynamics_heads(x, c.reward_logits, c.reward, c.hidden, c.pool_hidden, c.pool_stride, c.out_slot)) return MZ_ECUDA;
    }
    const float* x = R.tower_tc(R.prediction_site(tc_tower_input(r, MZ_TOWER_PREDICTION)));
    if (!x) return MZ_ECUDA;
    if (!R.prediction_heads(x, c.value_logits, c.policy_logits, c.value)) return MZ_ECUDA;
    return MZ_OK;
}

int resnet_state_elems(const ResNetDevice* r) { return state_elems(r); }
bool resnet_uses_tensor_cores(const ResNetDevice* r) { return is_tc(r->route); }

// Partitioned replay (abi.cu) needs every kernel of a recurrent inference to honour a first-game offset: the x3 towers,
// the fused small towers and heads_kernel do; the per-layer convs, the fp16-mode towers and the generic heads route do not.
static const int32_t kDryRunAction = 0;        // stands for the action array in dry runs (only its presence matters)
bool resnet_can_partition(const ResNetDevice* r0) {
    ResNetDevice* r = const_cast<ResNetDevice*>(r0);
    if (!r->loaded) return false;
    if (is_tc(r->route)) return r->route == TowerRoute::TcX3;
    std::string err; int64_t launches = 0;
    Runner R{r, nullptr, &launches, &err, r->max_batch, 0};
    if (r->net.blocks < 1) return false;
    // the wide towers honour g0 (resnet_create accepted the board); otherwise the fused small towers must take both towers
    if (!is_wide(r->route) && R.small_tower(R.dynamics_site(nullptr, &kDryRunAction), nullptr, true) != 1) return false;
    if (!is_wide(r->route) && R.small_tower(R.prediction_site(nullptr), nullptr, true) != 1) return false;
    // heads_kernel route (not heads_big): the weights of all three heads plus one group's tile fit in shared memory
    const HeadDesc* hs[3] = {&r->reward_head, &r->value_head, &r->policy_head};
    return heads_fit_one_group(heads_footprint(r->C, r->hh * r->hw, 3, hs));
}
const char* resnet_numerics(const ResNetDevice* r) {
    switch (r->route) {
    case TowerRoute::Wide256:
        return "f32-grade nets (256-channel towers on the tensor cores, output channels split across CTA pairs, split fp16 "
               "operands x = x_h + x_l/2^11, 3 partial products, f32 accumulate; f32 stems and heads) + f64 tree statistics";
    case TowerRoute::WidePair:
        return "f32-grade nets (128-channel towers on the tensor cores, boards split across CTA pairs, split fp16 operands "
               "x = x_h + x_l/2^11, 3 partial products, f32 accumulate; f32 stems and heads) + f64 tree statistics";
    case TowerRoute::Wide:
        return "f32-grade nets (128-channel towers on the tensor cores, split fp16 operands x = x_h + x_l/2^11, 3 partial "
               "products, f32 accumulate; f32 stems and heads) + f64 tree statistics";
    case TowerRoute::TcX3:
        return "f32-grade nets (tensor-core towers on split fp16 operands x = x_h + x_l/2^11, 3 partial products, f32 accumulate; f32 heads) + f64 tree statistics";
    case TowerRoute::TcF16: return "fp16 operands / f32 accumulate (tensor-core towers), f32 heads, f64 tree statistics";
    case TowerRoute::CudaCore: break;
    }
    return r->note.empty() ? "f32 nets + f64 tree statistics" : r->note.c_str();
}

// Range guard of the x3 towers: number of epilogue threads that stored an activation beyond the fp16 range since the
// last call (synchronises the stream).  resnet_use_strict switches the handle to the fp32 CUDA-core towers for good.
int resnet_take_saturations(ResNetDevice* r, cudaStream_t stream) {
    if (!range_guarded(r->route) || !r->d_sat) return 0;
    int count = 0;
    if (cudaMemcpyAsync(&count, r->d_sat, 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess) return 0;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return 0;
    if (count) cudaMemsetAsync(r->d_sat, 0, 4, stream);
    return count;
}
void resnet_use_strict(ResNetDevice* r) {
    r->note = r->route == TowerRoute::Wide256
                  ? "f32 nets + f64 tree statistics (256-channel tensor-core towers left after an activation exceeded the fp16 range)"
              : is_wide(r->route)
                  ? "f32 nets + f64 tree statistics (128-channel tensor-core towers left after an activation exceeded the fp16 range)"
                  : "f32 nets + f64 tree statistics (tensor-core towers left after an activation exceeded the fp16 range)";
    r->route = TowerRoute::CudaCore;                 // dense NCHW states: smaller than the board layout, the pool fits
}

// Launch plan of conv3x3_kernel for a shape (host only, behind mz_debug_conv3x3_plan): plan[12] = {P, stride, MAX_ITEMS,
// bands, band_rows, boards per CTA, cin chunk, grid x, grid y, grid z, shared-memory bytes, cout tile}.
bool resnet_conv_plan(int n, int cin, int cout, int H, int W, int stride, int64_t* plan, std::string* err) {
    ConvPlan p;
    if (!conv3x3_plan(n, cin, cout, H, W, stride, &p, err)) return false;
    const int64_t out[12] = {p.P, p.stride, p.max_items, p.bands, p.band_rows, p.boards, p.cin_chunk,
                             p.grid.x, p.grid.y, p.grid.z, (int64_t)p.smem, p.cout_tile};
    for (int i = 0; i < 12; ++i) plan[i] = out[i];
    return true;
}

// A synthetic net of plain convs for the debug entries: the state_dict "c<i>.weight" of n_convs convs whose OIHW weights
// follow one another in `w` (conv i reads cin[i] planes), packed as `route` packs its towers, with bias[i] (cout floats
// each) when biases are given.
static bool pack_debug_convs(TowerRoute route, int n_convs, const int* cin, int cout, int stride, int H, int W, const float* w,
                             const float* bias, std::vector<float>& blob, std::vector<ConvLayer>& layers, std::string* err) {
    std::vector<std::string> names(n_convs);
    std::vector<MzTensor> tensors(n_convs);
    size_t w_off = 0;
    for (int i = 0; i < n_convs; ++i) {
        names[i] = "c" + std::to_string(i) + ".weight";
        tensors[i] = MzTensor{names[i].c_str(), w + w_off, (int64_t)cout * cin[i] * 9};
        w_off += (size_t)cout * cin[i] * 9;
    }
    Loader L{tensors.data(), n_convs, err};
    for (int i = 0; i < n_convs; ++i) {
        if (!pack_conv(L, "c" + std::to_string(i), "", cin[i], cout, stride, blob, layers, weight_image(route), H, W)) return false;
        if (bias) {
            layers.back().b_off = (long)blob.size();
            blob.insert(blob.end(), bias + (size_t)i * cout, bias + (size_t)(i + 1) * cout);      // (cout % 4 == 0: stays aligned)
        }
    }
    return true;
}

// Stand-alone conv3x3 (+bias, +residual, +ReLU) on host NCHW data through either implementation.
// Debug / parity entry point behind mz_debug_conv3x3.  The CUDA-core kernel takes any cin, cout (a multiple of 4) and
// stride 1 or 2; the tensor-core convs take 64 -> 64 at stride 1 on their boards only.
int resnet_debug_conv(int n, int cin, int cout, int H, int W, int stride, const float* x, const float* w_oihw, const float* bias,
                      const float* residual, int relu, int use_tc, float* out, int sm_count, std::string* err) {
    if (use_tc && (cin != cout || stride != 1 || !conv_tc_supported(cout, H, W))) {
        *err = "shape not supported by the tensor-core conv"; return MZ_EUNSUPPORTED;
    }
    ConvPlan plan;
    if (!conv3x3_plan(n, cin, cout, H, W, stride, &plan, err)) return MZ_EINVAL;
    const int C = cout, Ho = conv_out(H, stride), Wo = conv_out(W, stride);
    MzNetDesc nd{};
    nd.kind = MZ_NET_RESNET; nd.channels = C; nd.obs_c = cin; nd.obs_h = H; nd.obs_w = W; nd.action_space = 1;
    ResNetDevice r{};
    r.net = nd; r.max_batch = n; r.sm_count = sm_count; r.C = C; r.hh = Ho; r.hw = Wo;
    r.route = use_tc == 2 ? TowerRoute::TcX3 : use_tc ? TowerRoute::TcF16 : TowerRoute::CudaCore;
    std::vector<float> blob;
    std::vector<ConvLayer> layers;
    if (!pack_debug_convs(r.route, 1, &cin, cout, stride, H, W, w_oihw, bias, blob, layers, err)) return MZ_EINVAL;
    const bool split = r.route == TowerRoute::TcX3;
    const size_t dense_in = (size_t)n * cin * H * W, dense = (size_t)n * C * Ho * Wo, packed = (size_t)n * conv_tc_board_elems(split);
    float *d_blob = nullptr, *d_x = nullptr, *d_res = nullptr, *d_out = nullptr, *d_px = nullptr, *d_pres = nullptr, *d_pout = nullptr;
    auto cleanup = [&]() { for (float* p : {d_blob, d_x, d_res, d_out, d_px, d_pres, d_pout}) if (p) cudaFree(p); };
    bool ok = cudaMalloc(&d_blob, blob.size() * 4) == cudaSuccess && cudaMalloc(&d_x, dense_in * 4) == cudaSuccess &&
              cudaMalloc(&d_out, dense * 4) == cudaSuccess && (!residual || cudaMalloc(&d_res, dense * 4) == cudaSuccess);
    if (ok && use_tc)
        ok = cudaMalloc(&d_px, packed * 4) == cudaSuccess && cudaMalloc(&d_pout, packed * 4) == cudaSuccess &&
             (!residual || cudaMalloc(&d_pres, packed * 4) == cudaSuccess);
    if (!ok) { cleanup(); *err = "allocation failed"; return MZ_ENOMEM; }
    cudaMemcpy(d_blob, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_x, x, dense_in * 4, cudaMemcpyHostToDevice);
    if (residual) cudaMemcpy(d_res, residual, dense * 4, cudaMemcpyHostToDevice);
    cudaMemset(d_out, 0xFF, dense * 4);                 // NaN: an output element the kernel does not write cannot pass a test
    r.d_conv = d_blob;
    int64_t launches = 0;
    Runner R{&r, nullptr, &launches, err, n};
    bool good;
    if (use_tc) {
        const unsigned blocks = (unsigned)((dense + 255) / 256);
        cudaMemset(d_px, 0, packed * 4);
        nchw_to_p64c4_kernel<<<blocks, 256>>>(d_x, d_px, n, C, H, W, split ? 1 : 0);
        if (residual) { cudaMemset(d_pres, 0, packed * 4); nchw_to_p64c4_kernel<<<blocks, 256>>>(d_res, d_pres, n, C, H, W, split ? 1 : 0); }
        good = R.conv_tc(layers[0], d_px, d_pout, residual ? d_pres : nullptr, relu != 0);
        if (good) p64c4_to_nchw_kernel<<<blocks, 256>>>(d_pout, d_out, n, C, H, W, split ? 1 : 0);
    } else {
        good = R.conv(layers[0], d_x, d_out, residual ? d_res : nullptr, relu != 0, H, W);
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (good && e != cudaSuccess) { good = false; *err = std::string("debug conv: ") + cudaGetErrorString(e); }
    // optional warm-L2 timing of the bare kernel: MZ_DEBUG_CONV_REPS=k prints the mean of k back-to-back launches
    const char* reps_env = getenv("MZ_DEBUG_CONV_REPS");
    if (good && reps_env && atoi(reps_env) > 0) {
        const int reps = atoi(reps_env);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0);
        for (int i = 0; i < reps; ++i) {
            if (use_tc) R.conv_tc(layers[0], d_px, d_pout, residual ? d_pres : nullptr, relu != 0);
            else R.conv(layers[0], d_x, d_out, residual ? d_res : nullptr, relu != 0, H, W);
        }
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        const double flops = 2.0 * n * Ho * Wo * (double)cin * cout * 9;
        fprintf(stderr, "[mz_debug_conv3x3] %s n=%d %d->%d %dx%d stride %d residual=%d: %.2f us per launch, %.1f TFLOP/s useful\n",
                use_tc ? "wgmma" : "cuda-core", n, cin, cout, H, W, stride, residual ? 1 : 0, 1000.0 * ms / reps,
                flops / (ms / reps * 1e-3) / 1e12);
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    if (good) cudaMemcpy(out, d_out, dense * 4, cudaMemcpyDeviceToHost);
    r.d_conv = nullptr;
    cleanup();
    return good ? MZ_OK : MZ_ECUDA;
}

// Stand-alone DownSample stem on host NCHW data, behind mz_debug_downsample: the network's packer (pack_downsample) and
// Runner::downsample.  w holds the 18 convs' [cout][cin][3][3] weights in execution order (conv1; resblocks1.0.conv1,
// .conv2, resblocks1.1.conv1, .conv2; conv2; resblocks2.0 ... 2; resblocks3.0 ... 2), bias their [cout] biases in the
// same order; conv1's and conv2's must be zero (the reference's have none).  Every device buffer but the input starts
// as NaN bytes (0xFF), so a stage that reads a plane nobody wrote produces NaN.
int resnet_debug_downsample(int n, int in, int C, int H, int W, const float* x, const float* w, const float* bias, float* out,
                            float* stages, int sm_count, std::string* err) {
    if (n < 1 || in < 1 || H < 1 || W < 1 || C < 8 || C % 8) { *err = "bad shape (C a positive multiple of 8)"; return MZ_EINVAL; }
    if (!plan_shapes(n, downsample_shapes(in, C, H, W), err)) return MZ_EUNSUPPORTED;
    // the state_dict of the stem under the prefix "d", one bias per conv
    std::vector<std::string> names;
    std::vector<int> cins, couts;
    auto add = [&](const std::string& s, int ci, int co) { names.push_back(s); cins.push_back(ci); couts.push_back(co); };
    add("d.conv1", in, C / 2);
    for (int i = 0; i < 2; ++i)
        for (int k = 1; k <= 2; ++k) add("d.resblocks1." + std::to_string(i) + ".conv" + std::to_string(k), C / 2, C / 2);
    add("d.conv2", C / 2, C);
    for (const std::string s : {"d.resblocks2.", "d.resblocks3."})
        for (int i = 0; i < 3; ++i)
            for (int k = 1; k <= 2; ++k) add(s + std::to_string(i) + ".conv" + std::to_string(k), C, C);
    const size_t n_convs = names.size();
    std::vector<std::string> keys;
    keys.reserve(2 * n_convs);                          // (c_str() of each key must stay put)
    std::vector<MzTensor> tensors;
    size_t w_off = 0, b_off = 0;
    for (size_t i = 0; i < n_convs; ++i) {
        if ((i == 0 || i == 5) && std::any_of(bias + b_off, bias + b_off + couts[i], [](float b) { return b != 0.0f; })) {
            *err = "conv1 and conv2 have no bias"; return MZ_EINVAL;
        }
        keys.push_back(names[i] + ".weight");
        tensors.push_back(MzTensor{keys.back().c_str(), w + w_off, (int64_t)couts[i] * cins[i] * 9});
        keys.push_back(names[i] + ".bias");
        tensors.push_back(MzTensor{keys.back().c_str(), bias + b_off, (int64_t)couts[i]});
        w_off += (size_t)couts[i] * cins[i] * 9;
        b_off += couts[i];
    }
    ResNetDevice r{};
    r.net.kind = MZ_NET_RESNET; r.net.channels = C; r.net.obs_c = in; r.net.obs_h = H; r.net.obs_w = W;
    r.net.action_space = 1; r.net.downsample = 1;
    r.max_batch = n; r.sm_count = sm_count; r.C = C; r.hh = (H + 15) / 16; r.hw = (W + 15) / 16;
    std::vector<float> blob;
    Loader L{tensors.data(), (int)tensors.size(), err};
    if (!pack_downsample(L, "d", in, C, false, blob, r.rep_down) || !L.ok) return MZ_EINVAL;

    const int h1 = conv_out(H, 2), w1 = conv_out(W, 2), h2 = conv_out(h1, 2), w2 = conv_out(w1, 2);
    const size_t half = (size_t)n * (C / 2) * h1 * w1, full = (size_t)n * C * h2 * w2;
    const size_t pooled = (size_t)n * C * conv_out(h2, 2) * conv_out(w2, 2), dense = (size_t)n * C * r.hh * r.hw;
    const size_t stage_elems[6] = {half, half, full, full, pooled, pooled};
    float *d_blob = nullptr, *d_x = nullptr, *d_stage[6] = {};
    auto cleanup = [&]() {
        for (float* p : {d_blob, d_x, r.ws[0], r.ws[1], r.ws[2]}) if (p) cudaFree(p);
        for (float* p : d_stage) if (p) cudaFree(p);
    };
    auto alloc = [](float** p, size_t floats) { return cudaMalloc(p, floats * 4 + 64) == cudaSuccess && cudaMemset(*p, 0xFF, floats * 4 + 64) == cudaSuccess; };
    bool ok = alloc(&d_blob, blob.size()) && alloc(&d_x, (size_t)n * in * H * W);
    for (int i = 0; ok && i < 3; ++i) ok = alloc(&r.ws[i], std::max(half, full));
    for (int i = 0; ok && stages && i < 6; ++i) ok = alloc(&d_stage[i], stage_elems[i]);
    if (!ok) { cleanup(); *err = "allocation failed"; return MZ_ENOMEM; }
    cudaMemcpy(d_blob, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_x, x, (size_t)n * in * H * W * 4, cudaMemcpyHostToDevice);
    r.d_conv = d_blob;
    int64_t launches = 0;
    Runner R{&r, nullptr, &launches, err, n};
    if (stages) R.ds_stages = d_stage;
    float *cur = r.ws[0], *tmp = r.ws[1], *spare = r.ws[2];
    bool good = R.downsample(d_x, &cur, &tmp, &spare);
    cudaError_t e = cudaDeviceSynchronize();
    if (good && e == cudaSuccess) e = cudaMemcpy(out, cur, dense * 4, cudaMemcpyDeviceToHost);
    for (int i = 0; good && stages && i < 6 && e == cudaSuccess; stages += stage_elems[i], ++i)
        e = cudaMemcpy(stages, d_stage[i], stage_elems[i] * 4, cudaMemcpyDeviceToHost);
    if (good && e != cudaSuccess) { good = false; *err = std::string("debug downsample: ") + cudaGetErrorString(e); }
    r.d_conv = nullptr;
    cleanup();
    return good ? MZ_OK : MZ_ECUDA;
}

// Launch plan of the fused CUDA-core tower (host only, behind mz_debug_small_tower_plan): plan[6] = {P, CO, boards per
// CTA, threads, grid, shared-memory bytes} of n boards through [a stem conv reading in_channels planes +] `blocks`
// residual blocks of C channels, from the same Runner::small_tower_args and planner the launch takes.  false with the
// reason in *err when the fused tower refuses the shape (the network then runs one conv3x3_kernel launch per conv).
bool resnet_small_tower_plan(int n, int in_channels, int C, int H, int W, int blocks, bool stem, int sm_count, int64_t* plan,
                             std::string* err) {
    if (blocks < 0 || in_channels < 1) { *err = "bad shape"; return false; }
    if (!stem && in_channels != C) { *err = "without a stem the tower input has C channels"; return false; }
    if ((stem ? 1 : 0) + 2 * blocks < 1 || (stem ? 1 : 0) + 2 * blocks > kSmallTowerMaxLayers) { *err = "1 to 10 layers"; return false; }
    ResNetDevice r{};
    r.C = C; r.hh = H; r.hw = W; r.sm_count = sm_count; r.net.action_space = 1; r.net.blocks = blocks;
    std::vector<ConvLayer> layers((stem ? 1 : 0) + 2 * (size_t)blocks);
    for (size_t i = 0; i < layers.size(); ++i) {
        ConvLayer& l = layers[i];
        l.cin = stem && i == 0 ? in_channels : C; l.cout = C; l.stride = 1;
        l.w_off = 0; l.b_off = -1; l.tc_off = l.tc_table_off = l.tc_scale_off = -1;
    }
    int64_t launches = 0;
    Runner R{&r, nullptr, &launches, err, n};
    SmallTowerArgs a{};
    if (!R.small_tower_args(a, TowerSite{&layers, 0, stem, in_channels, H, W, nullptr, nullptr, 0, nullptr}, nullptr)) {
        *err = "layers the fused tower does not take"; return false;
    }
    SmallTowerPlan p;
    const char* why = "";
    if (!small_tower_plan(a, sm_count, &p, &why)) { *err = why; return false; }
    const int64_t out[6] = {p.P, p.CO, p.boards_per_cta, p.threads, p.grid, (int64_t)p.smem};
    for (int i = 0; i < 6; ++i) plan[i] = out[i];
    return true;
}

// Launch plan of the wide tower (host only, behind mz_debug_wide_tower_plan): plan[9] = {M-tiles, threads, shared-memory bytes,
// weight ring stages, layers, CTAs per SM, boards per wave, launches, registers per thread assumed} of n boards of C x H x W
// through [a stem conv +] `blocks` residual blocks.  false with the reason in *err when the wide towers refuse the shape.
// With `pair`, the plan of the CTA-pair tower (mz_debug_wide_pair_tower_plan): plan[9] = {board rows of CTA 0, M-tiles per
// CTA, threads per CTA, shared-memory bytes per CTA, weight ring stages, layers, boards (clusters) per wave, launches,
// registers per thread assumed}.
static void wide_plan_export(const WideTowerPlan& p, bool pair, int64_t* plan) {
    const int64_t one[9] = {p.m_tiles, p.threads, (int64_t)p.smem, p.stages, p.layers, p.ctas_per_sm, p.wave, p.launches, p.reg_cap};
    const int64_t two[9] = {p.pair_rows0, p.m_tiles, p.threads, (int64_t)p.smem, p.stages, p.layers, p.wave, p.launches, p.reg_cap};
    for (int i = 0; i < 9; ++i) plan[i] = pair ? two[i] : one[i];
}
bool resnet_wide_tower_plan(int n, int C, int H, int W, int blocks, bool stem, int sm_count, int64_t* plan, std::string* err,
                            bool pair) {
    if (blocks < 0) { *err = "bad shape"; return false; }
    WideTowerPlan p;
    const char* why = "";
    if (!(pair ? wide_pair_plan : wide_tower_plan)(n, C, H, W, (stem ? 1 : 0) + 2 * blocks, sm_count, &p, &why)) { *err = why; return false; }
    wide_plan_export(p, pair, plan);
    return true;
}

// Launch plan of the 256-channel tower (host only, behind mz_debug_wide256_tower_plan): plan[10] = {boards per CTA pair,
// M-tiles per CTA, threads per CTA, shared-memory bytes per CTA, weight ring stages, layers, CTAs per SM, boards per wave,
// launches, registers per thread assumed}.  force_boards > 0 plans that many boards per CTA pair.
static void wide256_plan_export(const Wide256Plan& p, int64_t* plan) {
    const int64_t v[10] = {p.boards, p.m_tiles, p.threads, (int64_t)p.smem, p.stages, p.layers, p.ctas_per_sm, p.wave,
                           p.launches, p.reg_cap};
    for (int i = 0; i < 10; ++i) plan[i] = v[i];
}
bool resnet_wide256_tower_plan(int n, int C, int H, int W, int blocks, bool stem, int sm_count, int force_boards, int64_t* plan,
                               std::string* err) {
    if (blocks < 0) { *err = "bad shape"; return false; }
    Wide256Plan p;
    const char* why = "";
    if (!wide256_plan(n, C, H, W, (stem ? 1 : 0) + 2 * blocks, sm_count, force_boards, &p, &why)) { *err = why; return false; }
    wide256_plan_export(p, plan);
    return true;
}

// Stand-alone tower of one call site of the network, through the same site descriptions, Runner helpers and weight
// packing, on host NCHW data: a 64-channel tensor-core tower of resnet_inference_tc (TcF16 / TcX3, the input staged in
// the board layout where that function leaves it), the fused CUDA-core tower (CudaCore) or a wide tower (Wide / WidePair)
// of resnet_inference.  The workspaces, the prediction site's scratch state, the pool and the output start as NaN bytes
// (0xFF); only the input boards are written, with the zero padding the board layout promises.  So a layer that reads a
// board, a padding row or a pool slot nobody wrote produces NaN.
int resnet_debug_tower(TowerRoute route, int n, int in_channels, int C, int H, int W, int blocks, int site, int parts, int A,
                       const float* x, const float* w, const float* bias, const int32_t* action, const int32_t* parent,
                       int pool_stride, float* out, int64_t* launches, int32_t* saturated, int64_t* plan, int sm_count,
                       std::string* err, int force_boards) {
    const bool tc = is_tc(route), fused = route == TowerRoute::CudaCore, pair = route == TowerRoute::WidePair;
    const bool w256 = route == TowerRoute::Wide256;
    const bool dyn = site == MZ_TOWER_DYNAMICS || site == MZ_TOWER_DYNAMICS_POOL;
    const bool in_pool = site == MZ_TOWER_DYNAMICS_POOL;
    // only the fused tower takes the representation stem: the others leave it to conv3x3_kernel
    const bool stem = dyn || (fused && site == MZ_TOWER_REPRESENTATION);
    if (n < 1 || blocks < 0 || (!stem && blocks < 1) || site < MZ_TOWER_REPRESENTATION || site > MZ_TOWER_PREDICTION ||
        (fused && (C < 4 || (site == MZ_TOWER_REPRESENTATION ? in_channels < 1 : in_channels != C))) ||
        (tc && !conv_tc_supported(C, H, W))) {
        *err = tc ? "bad shape, site or mode" : "bad shape or site"; return MZ_EINVAL;
    }
    if (parts < 1 || parts > 4 || (parts > 1 && (!in_pool || route == TowerRoute::TcF16))) {
        *err = tc ? "partitions need the x3 towers at the in-search dynamics site, 1 to 4 of them"
                  : "partitions need the in-search dynamics site, 1 to 4 of them";
        return MZ_EINVAL;
    }
    if (dyn) {
        if (A < 1 || !action) { *err = "the dynamics sites need actions and A >= 1"; return MZ_EINVAL; }
        for (int g = 0; g < n; ++g) if (action[g] < 0 || action[g] >= A) { *err = "action out of range"; return MZ_EINVAL; }
    }
    if (in_pool) {
        if (!parent || pool_stride < 1) { *err = "the in-search site needs parents and pool_stride >= 1"; return MZ_EINVAL; }
        for (int g = 0; g < n; ++g) if (parent[g] < 0 || parent[g] >= pool_stride) { *err = "parent out of range"; return MZ_EINVAL; }
    }
    if (w256) {
        int64_t unused[10];
        std::string why;
        if (!resnet_wide256_tower_plan(n, C, H, W, blocks, stem, sm_count, force_boards, unused, &why)) {
            *err = "the 256-channel tower refuses the shape: " + why; return MZ_EUNSUPPORTED;
        }
    } else if (is_wide(route)) {
        int64_t unused[9];
        std::string why;
        if (!resnet_wide_tower_plan(n, C, H, W, blocks, stem, sm_count, unused, &why, pair)) {
            *err = std::string(pair ? "the wide pair tower" : "the wide tower") + " refuses the shape: " + why; return MZ_EUNSUPPORTED;
        }
    }
    // the site's convs, the stem first: [C][in_channels or C + 1][3][3], then two [C][C][3][3] per block
    const int n_convs = (stem ? 1 : 0) + 2 * blocks;
    std::vector<int> cin(n_convs, C);
    if (stem) cin[0] = dyn ? C + 1 : in_channels;
    MzNetDesc nd{};
    nd.kind = MZ_NET_RESNET; nd.channels = C; nd.obs_c = site == MZ_TOWER_REPRESENTATION ? in_channels : C; nd.obs_h = H;
    nd.obs_w = W; nd.action_space = dyn ? A : 1; nd.blocks = blocks;
    ResNetDevice r{};
    r.net = nd; r.max_batch = n; r.sm_count = sm_count; r.C = C; r.hh = H; r.hw = W; r.route = route;
    std::vector<float> blob;
    std::vector<ConvLayer> layers;
    if (!pack_debug_convs(route, n_convs, cin.data(), C, 1, H, W, w, bias, blob, layers, err)) return MZ_EINVAL;
    if (site == MZ_TOWER_REPRESENTATION) {
        r.rep_trunk = layers;
        if (!stem) r.rep_trunk.insert(r.rep_trunk.begin(), ConvLayer{});      // [0]: the CUDA-core stem, not run here
    } else if (dyn) {
        r.dyn = layers;
    } else {
        r.pred = layers;
    }

    // one stored input board: the tensor-core board layout, or dense planes
    const size_t in_elems = (size_t)nd.obs_c * H * W, dense = (size_t)n * C * H * W;
    const size_t board = tc ? (size_t)conv_tc_board_elems(route == TowerRoute::TcX3) : in_elems, boards = (size_t)n * board;
    const size_t pool_floats = in_pool ? (size_t)n * pool_stride * board : 0;
    float *d_blob = nullptr, *d_x = nullptr, *d_stage = nullptr, *d_out = nullptr, *d_pool = nullptr;
    int32_t *d_action = nullptr, *d_parent = nullptr;
    auto cleanup = [&]() {
        for (void* p : {(void*)d_blob, (void*)d_x, (void*)d_stage, (void*)d_out, (void*)d_pool, (void*)d_action, (void*)d_parent,
                        (void*)r.ws[0], (void*)r.ws[1], (void*)r.ws[2], (void*)r.scratch_state, (void*)r.d_sat})
            if (p) cudaFree(p);
        r.ws[0] = r.ws[1] = r.ws[2] = r.scratch_state = nullptr; r.d_sat = nullptr; r.d_conv = nullptr;
    };
    bool ok = cudaMalloc(&d_blob, blob.size() * 4) == cudaSuccess && cudaMalloc(&d_x, (size_t)n * in_elems * 4) == cudaSuccess &&
              cudaMalloc(&d_stage, boards * 4) == cudaSuccess && cudaMalloc(&d_out, dense * 4) == cudaSuccess &&
              cudaMalloc(&r.scratch_state, boards * 4) == cudaSuccess && cudaMalloc(&r.d_sat, 64) == cudaSuccess &&
              cudaMalloc(&d_action, (size_t)n * 4) == cudaSuccess && cudaMalloc(&d_parent, (size_t)n * 4) == cudaSuccess &&
              (!in_pool || cudaMalloc(&d_pool, pool_floats * 4) == cudaSuccess);
    for (int i = 0; ok && i < 3; ++i) ok = cudaMalloc(&r.ws[i], boards * 4) == cudaSuccess;
    if (!ok) { cleanup(); *err = "allocation failed"; return MZ_ENOMEM; }
    r.d_conv = d_blob;
    cudaMemcpy(d_blob, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_x, x, (size_t)n * in_elems * 4, cudaMemcpyHostToDevice);
    if (dyn) cudaMemcpy(d_action, action, (size_t)n * 4, cudaMemcpyHostToDevice);
    if (in_pool) cudaMemcpy(d_parent, parent, (size_t)n * 4, cudaMemcpyHostToDevice);
    for (int i = 0; i < 3; ++i) cudaMemset(r.ws[i], 0xFF, boards * 4);
    cudaMemset(r.scratch_state, 0xFF, boards * 4);
    cudaMemset(d_out, 0xFF, dense * 4);
    cudaMemset(r.d_sat, 0, 64);
    // the input boards, zero padded, where the stage before the tower leaves them
    const unsigned cblocks = (unsigned)((dense + 255) / 256);
    const float* stage = d_x;
    if (tc) {
        cudaMemset(d_stage, 0, boards * 4);
        nchw_to_p64c4_kernel<<<cblocks, 256>>>(d_x, d_stage, n, C, H, W, route == TowerRoute::TcX3);
        stage = d_stage;
    }
    const float* in = stage;
    if (in_pool) {
        cudaMemset(d_pool, 0xFF, pool_floats * 4);
        for (int g = 0; g < n; ++g)
            cudaMemcpy(d_pool + ((size_t)g * pool_stride + parent[g]) * board, stage + (size_t)g * board, board * 4,
                       cudaMemcpyDeviceToDevice);
        in = d_pool;
    } else if (tc) {
        float* dst = tc_tower_input(&r, site);
        cudaMemcpy(dst, stage, boards * 4, cudaMemcpyDeviceToDevice);
        in = dst;
    }
    int64_t n_launches = 0;
    SmallTowerPlan small_used{}, small_first{};
    WideTowerPlan wide_used{}, wide_first{};
    Wide256Plan w256_used{}, w256_first{};
    const float* result = nullptr;
    int rc = MZ_OK;
    // the ranges of the partitioned replay, each through its own Runner (one range unless in the pool); every array stays
    // addressed by the global game.  The plan reported is the first range's.
    const int per = in_pool ? partition_games(n, parts) : n;
    for (int p = 0; p * per < n && rc == MZ_OK; ++p) {
        Runner R{&r, nullptr, &n_launches, err, std::min(per, n - p * per), p * per};
        R.small_plan = &small_used; R.wide_plan_out = &wide_used; R.wide256_plan_out = &w256_used;
        R.wide256_boards = force_boards;
        const TowerSite s = site == MZ_TOWER_REPRESENTATION ? R.representation_site(in, !stem)
                          : site == MZ_TOWER_PREDICTION     ? R.prediction_site(in)
                          : R.dynamics_site(in, d_action, in_pool ? d_parent : nullptr, in_pool ? pool_stride : 0);
        const float* res = d_out;
        if (tc) {
            res = R.tower_tc(s);
            if (!res) rc = MZ_ECUDA;
        } else {
            const int done = fused ? R.small_tower(s, d_out) : R.wide_tower(s, d_out);
            if (done < 0) {
                rc = MZ_ECUDA;
            } else if (done == 0 && fused) {
                int64_t unused[6];
                std::string why = "no fused launch";
                resnet_small_tower_plan(R.n, stem ? cin[0] : C, C, H, W, blocks, stem, sm_count, unused, &why);
                *err = "the fused tower refuses the shape: " + why; rc = MZ_EUNSUPPORTED;
            } else if (done == 0) {
                *err = "no wide launch"; rc = MZ_EUNSUPPORTED;
            }
        }
        if (rc == MZ_OK && result && res != result) { *err = "partitions ended in different buffers"; rc = MZ_ECUDA; }
        result = res;
        if (p == 0) { small_first = small_used; wide_first = wide_used; w256_first = w256_used; }
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (rc == MZ_OK && e != cudaSuccess) { rc = MZ_ECUDA; *err = std::string("debug tower: ") + cudaGetErrorString(e); }
    if (rc == MZ_OK) {
        if (tc) p64c4_to_nchw_kernel<<<cblocks, 256>>>(result, d_out, n, C, H, W, route == TowerRoute::TcX3);
        int sat = 0;
        e = cudaMemcpy(out, d_out, dense * 4, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(&sat, r.d_sat, 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { rc = MZ_ECUDA; *err = std::string("debug tower: ") + cudaGetErrorString(e); }
        if (saturated) *saturated = sat;
        if (plan && fused) {
            const SmallTowerPlan& f = small_first;
            const int64_t pl[6] = {f.P, f.CO, f.boards_per_cta, f.threads, f.grid, (int64_t)f.smem};
            for (int i = 0; i < 6; ++i) plan[i] = pl[i];
        }
        if (plan && w256) wide256_plan_export(w256_first, plan);
        else if (plan && is_wide(route)) wide_plan_export(wide_first, pair, plan);
    }
    if (launches) *launches = n_launches;
    cleanup();
    return rc;
}

// The heads of one call site of the network as a ResNetDevice holds them: C channels on an H x W board, states in `layout`
// (kLayoutDense / kLayoutF16 / kLayoutSplit), head descriptors laid out as pack_head lays them from shapes[h] = {reduced
// channels, n_out, hidden layers, widths...}.  The representation site has no head, the dynamics sites the reward head,
// the prediction site the value and the policy head; the first head of a site is scalarised (n_out = 2 S + 1).
static bool debug_heads_device(ResNetDevice& r, int C, int H, int W, int site, int layout, const int32_t* shapes, int sm_count,
                               int* n_heads, std::string* err) {
    if (C < 4 || C % 4 || H < 1 || W < 1 || site < MZ_TOWER_REPRESENTATION || site > MZ_TOWER_PREDICTION ||
        layout < kLayoutDense || layout > kLayoutSplit) {
        *err = "bad shape, site or layout"; return false;
    }
    if (layout != kLayoutDense && (C != 64 || H > 6 || W > 7)) { *err = "the board layouts hold 64 channels on boards up to 6 x 7"; return false; }
    *n_heads = site == MZ_TOWER_REPRESENTATION ? 0 : site == MZ_TOWER_PREDICTION ? 2 : 1;
    if (*n_heads > 0 && !shapes) { *err = "head shapes missing"; return false; }
    r = ResNetDevice{};
    r.C = C; r.hh = H; r.hw = W; r.sm_count = sm_count; r.max_batch = 0;
    r.route = layout == kLayoutSplit ? TowerRoute::TcX3 : layout == kLayoutF16 ? TowerRoute::TcF16 : TowerRoute::CudaCore;
    HeadDesc* dst[2] = {site == MZ_TOWER_PREDICTION ? &r.value_head : &r.reward_head, &r.policy_head};
    size_t size = 0;
    for (int h = 0; h < *n_heads; ++h) {
        const int32_t* s = shapes + (size_t)h * (3 + MZ_MAX_LAYERS);
        bool ok = s[0] >= 1 && s[1] >= 1 && s[2] >= 0 && s[2] <= MZ_MAX_LAYERS;
        for (int l = 0; ok && l < s[2]; ++l) ok = s[3 + l] >= 1;
        if (!ok) { *err = "bad head shape"; return false; }
        if (h == 0 && s[1] % 2 == 0) { *err = "the scalarised head has 2 S + 1 logits"; return false; }
        layout_head(C, s[0], H * W, s + 3, s[2], s[1], &size, *dst[h]);
    }
    r.net.support_size = *n_heads > 0 ? shapes[1] / 2 : 0;
    return true;
}

// arguments of the heads launch of `site` (what the Runner helper of the site passes to Runner::heads)
static HeadsArgs debug_heads_args(Runner& R, int site, int n_heads) {
    ResNetDevice* r = R.r;
    const HeadDesc* h0 = site == MZ_TOWER_PREDICTION ? &r->value_head : &r->reward_head;
    return R.heads_args(nullptr, n_heads, n_heads > 0 ? h0 : nullptr, n_heads > 1 ? &r->policy_head : nullptr, nullptr, nullptr,
                        nullptr, nullptr, nullptr, nullptr, 0, 0);
}

// Launch plan of one heads call (host only, behind mz_debug_heads_plan): plan[5] = {route, groups per CTA, threads, grid,
// shared-memory bytes} of the samples [g0, g0 + n) from Runner::plan_heads, the planner the launch takes; false with the
// reason in *err when the shape or the forced route is refused.
bool resnet_heads_plan(int n, int g0, int C, int H, int W, int site, int layout, int route, const int32_t* shapes, int sm_count,
                       int64_t* plan, std::string* err) {
    if (n < 1 || g0 < 0 || route < MZ_HEADS_PLANNED || route > MZ_HEADS_GENERIC) { *err = "bad batch or route"; return false; }
    ResNetDevice r;
    int n_heads;
    if (!debug_heads_device(r, C, H, W, site, layout, shapes, sm_count, &n_heads, err)) return false;
    int64_t launches = 0;
    Runner R{&r, nullptr, &launches, err, n, g0};
    R.heads_route = route;
    HeadsPlan p;
    if (!R.plan_heads(debug_heads_args(R, site, n_heads), &p)) return false;
    const int64_t out[5] = {p.route, p.groups, p.threads, p.grid, (int64_t)p.smem};
    for (int i = 0; i < 5; ++i) plan[i] = out[i];
    return true;
}

// Stand-alone heads call of one call site of resnet_inference, through the same Runner helpers, on host NCHW data encoded
// into `layout`.  Every output starts as NaN bytes (0xFF): so do the pool's other slots and the board layouts' padding.
int resnet_debug_heads(int n, int C, int H, int W, int site, int layout, int route, int parts, const int32_t* shapes,
                       const MzTensor* tensors, int n_tensors, const float* x, int pool_stride, int out_slot, float* logits0,
                       float* logits1, float* scalar, float* rescaled, float* pool, float* state, int64_t* plan, int sm_count,
                       std::string* err) {
    ResNetDevice r;
    int n_heads;
    if (n < 1 || !debug_heads_device(r, C, H, W, site, layout, shapes, sm_count, &n_heads, err)) {
        if (n < 1) *err = "bad batch";
        return MZ_EINVAL;
    }
    const bool pooled = site != MZ_TOWER_PREDICTION;
    if (parts < 1 || parts > 4 || (parts > 1 && site != MZ_TOWER_DYNAMICS_POOL)) { *err = "partitions need the in-search dynamics site, 1 to 4 of them"; return MZ_EINVAL; }
    if (pooled && (pool_stride < 1 || out_slot < 0 || out_slot >= pool_stride)) { *err = "the rescaling sites need pool_stride >= 1 and 0 <= out_slot < pool_stride"; return MZ_EINVAL; }
    // pack the heads from the state_dict: "h<i>.conv.{weight,bias}", "h<i>.fc.<2l>.{weight,bias}"
    Loader L{tensors, n_tensors, err};
    std::vector<float> blob;
    HeadDesc* dst[2] = {site == MZ_TOWER_PREDICTION ? &r.value_head : &r.reward_head, &r.policy_head};
    for (int h = 0; h < n_heads; ++h) {
        const int32_t* s = shapes + (size_t)h * (3 + MZ_MAX_LAYERS);
        const std::string p = "h" + std::to_string(h);
        if (!pack_head(L, p + ".conv", p + ".fc", C, s[0], H * W, s + 3, s[2], s[1], blob, *dst[h])) return MZ_EINVAL;
    }
    // every range's plan first: a refused route is MZ_EUNSUPPORTED, not a failed launch
    const int per = site == MZ_TOWER_DYNAMICS_POOL ? partition_games(n, parts) : n;
    for (int g0 = 0; g0 < n; g0 += per) {
        int64_t unused[5];
        if (!resnet_heads_plan(std::min(per, n - g0), g0, C, H, W, site, layout, route, shapes, sm_count, unused, err)) return MZ_EUNSUPPORTED;
    }
    const size_t dense = (size_t)n * C * H * W;
    const size_t elems = layout != kLayoutDense ? (size_t)conv_tc_board_elems(layout == kLayoutSplit) : (size_t)C * H * W;
    const int n_out0 = n_heads > 0 ? shapes[1] : 0, n_out1 = n_heads > 1 ? shapes[3 + MZ_MAX_LAYERS + 1] : 0;
    float *d_blob = nullptr, *d_x = nullptr, *d_in = nullptr, *d_l0 = nullptr, *d_l1 = nullptr, *d_sc = nullptr, *d_resc = nullptr,
          *d_pool = nullptr, *d_state = nullptr;
    auto cleanup = [&]() {
        for (void* p : {(void*)d_blob, (void*)d_x, (void*)d_in, (void*)d_l0, (void*)d_l1, (void*)d_sc, (void*)d_resc, (void*)d_pool,
                        (void*)d_state, (void*)r.big_scratch})
            if (p) cudaFree(p);
    };
    auto alloc = [](float** p, size_t floats) { return cudaMalloc(p, floats * 4 + 64) == cudaSuccess && cudaMemset(*p, 0xFF, floats * 4 + 64) == cudaSuccess; };
    const bool ok = alloc(&d_blob, blob.size()) && alloc(&d_x, dense) && alloc(&d_in, (size_t)n * elems) && alloc(&d_l0, (size_t)n * n_out0) &&
                    alloc(&d_l1, (size_t)n * n_out1) && alloc(&d_sc, 2 * (size_t)n) && alloc(&d_resc, dense) &&
                    alloc(&d_pool, (size_t)n * std::max(pool_stride, 1) * elems) && alloc(&d_state, (size_t)n * elems);
    if (!ok) { cleanup(); *err = "allocation failed"; return MZ_ENOMEM; }
    cudaMemcpy(d_blob, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_x, x, dense * 4, cudaMemcpyHostToDevice);
    if (layout != kLayoutDense) {
        cudaMemset(d_in, 0, (size_t)n * elems * 4);                    // padding positions read as zero, as in the workspaces
        nchw_to_p64c4_kernel<<<(unsigned)((dense + 255) / 256), 256>>>(d_x, d_in, n, C, H, W, layout == kLayoutSplit);
    } else {
        cudaMemcpy(d_in, x, dense * 4, cudaMemcpyHostToDevice);
    }
    r.d_head = d_blob; r.scratch_state = d_state;
    int64_t launches = 0;
    HeadsPlan used{}, first{};
    bool good = true;
    for (int g0 = 0; g0 < n && good; g0 += per) {
        Runner R{&r, nullptr, &launches, err, std::min(per, n - g0), g0};
        R.heads_route = route; R.heads_plan_out = &used;
        if (site == MZ_TOWER_REPRESENTATION) good = R.representation_heads(d_in, d_resc, d_pool, pool_stride, out_slot);
        else if (site == MZ_TOWER_PREDICTION) good = R.prediction_heads(d_in, d_l0, d_l1, d_sc);
        else good = R.dynamics_heads(d_in, d_l0, d_sc, d_resc, d_pool, pool_stride, out_slot);
        if (g0 == 0) first = used;
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (good && e != cudaSuccess) { good = false; *err = std::string("debug heads: ") + cudaGetErrorString(e); }
    auto back = [&](float* host, const float* dev, size_t floats) {
        if (host && e == cudaSuccess) e = cudaMemcpy(host, dev, floats * 4, cudaMemcpyDeviceToHost);
    };
    if (good) {
        back(logits0, d_l0, (size_t)n * n_out0); back(logits1, d_l1, (size_t)n * n_out1); back(scalar, d_sc, 2 * (size_t)n);
        if (pooled) { back(rescaled, d_resc, dense); back(pool, d_pool, (size_t)n * pool_stride * elems); }
        if (pooled && layout != kLayoutDense) back(state, d_state, (size_t)n * elems);
        if (e != cudaSuccess) { good = false; *err = std::string("debug heads: ") + cudaGetErrorString(e); }
        const int64_t pl[5] = {first.route, first.groups, first.threads, first.grid, (int64_t)first.smem};
        if (plan) for (int i = 0; i < 5; ++i) plan[i] = pl[i];
    }
    r.d_head = nullptr; r.scratch_state = nullptr;
    cleanup();
    return good ? MZ_OK : MZ_ECUDA;
}

// stored hidden states (pool layout) -> dense NCHW, device to device
int resnet_states_to_nchw(ResNetDevice* r, const float* states, int count, float* out, cudaStream_t stream) {
    const size_t total = (size_t)count * r->C * r->hh * r->hw;
    if (is_tc(r->route))
        p64c4_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(states, out, count, r->C, r->hh, r->hw,
                                                                                   r->route == TowerRoute::TcX3);
    else cudaMemcpyAsync(out, states, total * 4, cudaMemcpyDeviceToDevice, stream);
    return cudaGetLastError() == cudaSuccess ? MZ_OK : MZ_ECUDA;
}

// dense NCHW states -> the pool layout, device to device (mz_import_tree)
int resnet_states_from_nchw(ResNetDevice* r, const float* dense, int count, float* states, cudaStream_t stream) {
    const size_t total = (size_t)count * r->C * r->hh * r->hw;
    if (is_tc(r->route)) {
        cudaMemsetAsync(states, 0, (size_t)count * state_elems(r) * 4, stream);          // padding positions read as zero
        nchw_to_p64c4_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dense, states, count, r->C, r->hh, r->hw,
                                                                                   r->route == TowerRoute::TcX3);
    } else {
        cudaMemcpyAsync(states, dense, total * 4, cudaMemcpyDeviceToDevice, stream);
    }
    return cudaGetLastError() == cudaSuccess ? MZ_OK : MZ_ECUDA;
}

// Fused search for small residual networks (small_search.cu): all the simulations of the games [c.g0, c.g0 + c.n) in ONE
// launch.  `c` is the recurrent call of the first simulation (pool mode), `tree` the tree step that follows it; the
// arguments of the towers and the heads are the ones resnet_inference would launch with, simulation after simulation.
static bool small_search_build(ResNetDevice* r, const InferCall& c, const TreeStepArgs& tree, int n_sims, SmallSearchArgs* out,
                               int* P, int* CO, int* G, int* threads, size_t* smem) {
    if (r->route != TowerRoute::CudaCore || !r->loaded || !r->fuse_small || !c.recurrent || !c.gather_parent || c.hidden || r->net.blocks < 1) return false;
    if (c.value_logits || c.reward_logits) return false;
    std::string err; int64_t launches = 0;
    Runner R{r, nullptr, &launches, &err, c.n, c.g0};
    const int C = r->C, hh = r->hh, hw = r->hw;
    SmallSearchArgs a{};
    float* raw = r->ws[0];                 // dynamics tower output
    float* pred_out = r->ws[1];            // prediction tower output
    float* hidden = r->scratch_hidden;     // rescaled state, dense (input of the prediction tower)
    if (!R.small_tower_args(a.dyn, R.dynamics_site(c.pool_hidden, c.action, c.gather_parent, c.pool_stride), raw)) return false;
    if (!R.small_tower_args(a.pred, R.prediction_site(hidden), pred_out)) return false;
    if (!small_tower_layout(a.dyn) || !small_tower_layout(a.pred)) return false;
    const int cap = std::max(a.dyn.cap_channels, a.pred.cap_channels);
    a.dyn.cap_channels = a.pred.cap_channels = cap;
    a.heads_dyn = R.heads_args(raw, 1, &r->reward_head, nullptr, nullptr, nullptr, c.reward, nullptr, nullptr, c.pool_hidden, c.pool_stride, c.out_slot);
    a.heads_pred = R.heads_args(pred_out, 2, &r->value_head, &r->policy_head, nullptr, c.policy_logits, c.value, nullptr, nullptr, nullptr, 0, 0);
    if (!(a.heads_dyn.C * a.heads_dyn.HW <= 1024)) return false;                   // one warp per sample (heads_kernel<32>)
    const int lo = std::min(a.heads_dyn.w_lo, a.heads_pred.w_lo);
    const int hi = std::max(a.heads_dyn.w_lo + a.heads_dyn.w_floats, a.heads_pred.w_lo + a.heads_pred.w_floats);
    a.heads_lo = lo & ~3; a.heads_floats = ((hi - a.heads_lo) + 3) & ~3;
    a.scratch_floats = std::max(a.heads_dyn.warp_floats, a.heads_pred.warp_floats);
    a.tree = tree;
    a.n = c.n; a.g0 = c.g0; a.n_sims = n_sims; a.first_slot = c.out_slot;
    int tile = 0, row_stride = 0, board_stride = 0;
    const int tower_floats = ((a.dyn.w_floats + 3) & ~3) + ((a.pred.w_floats + 3) & ~3);
    if (!small_search_shape(hh, hw, C, r->net.action_space, c.n, r->sm_count, tower_floats, a.heads_floats, a.scratch_floats, cap,
                            P, CO, G, &tile, threads, smem, &row_stride, &board_stride))
        return false;
    a.tile = tile;
    a.dyn.boards_per_cta = a.pred.boards_per_cta = tile;
    a.dyn.row_stride = a.pred.row_stride = row_stride;
    a.dyn.board_stride = a.pred.board_stride = board_stride;
    a.off_wd = 0;
    a.off_wp = (a.dyn.w_floats + 3) & ~3;
    a.off_wh = tower_floats;
    a.off_scratch = a.off_wh + a.heads_floats;
    a.off_map = a.off_scratch + (*threads / 32) * a.scratch_floats;
    a.off_act = a.off_map + 2 * C * hh * hw;
    *out = a;
    return true;
}

bool resnet_small_search_supported(ResNetDevice* r, const InferCall& c, const TreeStepArgs& tree, int n_sims) {
    // A/B switch: MZ_SMALL_SEARCH=0 keeps the step-wise pipeline, =1 uses the fused kernel wherever the shape allows
    constexpr bool kDefaultOn = true;
    const char* sw = getenv("MZ_SMALL_SEARCH");
    if (sw ? sw[0] != '1' : !kDefaultOn) return false;
    SmallSearchArgs a; int P, CO, G, threads; size_t smem;
    return small_search_build(r, c, tree, n_sims, &a, &P, &CO, &G, &threads, &smem);
}

int resnet_small_search(ResNetDevice* r, const InferCall& c, const TreeStepArgs& tree, int n_sims, cudaStream_t stream, int64_t* launches,
                        std::string* err) {
    SmallSearchArgs a; int P, CO, G, threads; size_t smem;
    if (!small_search_build(r, c, tree, n_sims, &a, &P, &CO, &G, &threads, &smem)) { *err = "small_search: shape not supported"; return MZ_EINVAL; }
    kt_begin(KT_SEARCH, stream);
    cudaError_t e = launch_small_search(a, P, CO, G, threads, smem, stream);
    kt_end(stream);
    if (e != cudaSuccess) { *err = std::string("small_search launch: ") + cudaGetErrorString(e); return MZ_ECUDA; }
    *launches += 1;
    return MZ_OK;
}

int resnet_inference(ResNetDevice* r, const InferCall& c, cudaStream_t stream, int64_t* launches, std::string* err) {
    if (!r->loaded) { *err = "weights not loaded"; return MZ_ESTATE; }
    if (c.g0 < 0 || c.g0 + c.n > r->max_batch) { *err = "batch larger than max_games"; return MZ_EINVAL; }
    if (is_tc(r->route)) return resnet_inference_tc(r, c, stream, launches, err);
    const MzNetDesc& nd = r->net;
    const int n = c.n, C = r->C, F = 2 * nd.support_size + 1;
    Runner R{r, stream, launches, err, n, c.g0};
    if (c.g0 != 0 && !c.recurrent) { *err = "resnet: partitioned calls are recurrent only"; return MZ_EINVAL; }
    float *cur = r->ws[0], *tmp = r->ws[1], *spare = r->ws[2];
    float* hidden_out = c.hidden ? c.hidden : r->scratch_hidden;
    const int kAll = Runner::kTryWide | Runner::kTryFused;

    if (!c.recurrent) {
        const float* x;
        if (nd.downsample == 2) {
            if (!R.cnn_stem(c.in, tmp, cur)) return MZ_ECUDA;
            x = R.site_tower(R.representation_site(cur), kAll, &cur, &tmp, &spare);
        } else if (nd.downsample) {
            if (!R.downsample(c.in, &cur, &tmp, &spare)) return MZ_ECUDA;
            // the stems stay on the CUDA cores; the trunk's blocks take the wide launch on the Wide256 route (the only
            // wide route that accepts a downsampled net)
            x = R.site_tower(R.representation_site(cur), kAll, &cur, &tmp, &spare);
        } else if (is_wide(r->route) && nd.blocks > 0) {
            // the stem on the CUDA cores, the blocks as one wide launch (per layer if the wide launch refuses)
            if (!R.conv(r->rep_trunk[0], c.in, cur, nullptr, true, nd.obs_h, nd.obs_w)) return MZ_ECUDA;
            x = R.site_tower(R.representation_site(cur, true), Runner::kTryWide, &cur, &tmp, &spare);
        } else {
            x = R.site_tower(R.representation_site(c.in), Runner::kTryFused, &cur, &tmp, &spare);
        }
        if (!x) return MZ_ECUDA;
        // rescale -> hidden (no heads on the raw state at the root)
        if (!R.representation_heads(x, hidden_out, c.pool_hidden, c.pool_stride, c.out_slot)) return MZ_ECUDA;
        if (c.reward_logits) {
            fill_root_reward_logits_kernel<<<(n * F + 255) / 256, 256, 0, stream>>>(c.reward_logits, n, F, nd.support_size);
            *launches += 1;
        }
        if (c.reward) {
            fill_root_reward_kernel<<<(n + 255) / 256, 256, 0, stream>>>(c.reward, n);
            *launches += 1;
        }
    } else {
        const TowerSite s = c.gather_parent ? R.dynamics_site(c.pool_hidden, c.action, c.gather_parent, c.pool_stride)
                                            : R.dynamics_site(c.in, c.action);
        const float* x = R.site_tower(s, kAll, &cur, &tmp, &spare);
        if (!x) return MZ_ECUDA;
        // reward head on the raw state + rescale -> hidden
        if (!R.dynamics_heads(x, c.reward_logits, c.reward, hidden_out, c.pool_hidden, c.pool_stride, c.out_slot)) return MZ_ECUDA;
    }
    // prediction on the rescaled state, which the tower reads and never writes
    const float* x = R.site_tower(R.prediction_site(hidden_out), kAll, &cur, &tmp, &spare);
    if (!x) return MZ_ECUDA;
    if (!R.prediction_heads(x, c.value_logits, c.policy_logits, c.value)) return MZ_ECUDA;
    return MZ_OK;
}

}  // namespace mz
