// Fully-connected MuZero networks evaluated by a group of G lanes for ONE sample.
//
// Device restatement of models.py:80-195 (MuZeroFullyConnectedNetwork) and models.py:630-642
// (mlp: Linear+ELU ... Linear+Identity) for inference:
//   representation  models.py:133-145   Linear stack, then per-sample min-max rescale
//   dynamics        models.py:147-170   [state | one_hot(action)] -> state', reward head on the
//                                       UN-normalised state', then rescale
//   prediction      models.py:128-131   policy head, value head
//   support_to_scalar models.py:645-666 fused behind the value / reward heads
// Weights live in shared memory as one blob: per Linear the transposed matrix [in][out]
// (lane o reads W[i*out+o]: consecutive lanes, consecutive banks) followed by the bias.
#pragma once
#include "common.cuh"
#include "../../include/mzb200.h"

namespace mz {

struct MlpDesc {
    int n;                               // number of Linear layers
    int in[MZ_MAX_LAYERS + 1];           // logical input width (for the dynamics net: dense part + |A|)
    int out[MZ_MAX_LAYERS + 1];
    int w_off[MZ_MAX_LAYERS + 1];        // float offset of the packed weights [ceil(in_dense/4)][out][4]
    int b_off[MZ_MAX_LAYERS + 1];        // float offset of bias [out]
    int in_dense[MZ_MAX_LAYERS + 1];     // rows that multiply the activation vector
    int x_off[MZ_MAX_LAYERS + 1];        // float offset of the one-hot rows [n_extra][out] (first layer of dynamics), or -1
};

struct FcNet {
    MlpDesc rep, dyn, rew, val, pol;
    int blob_floats;
    int obs_elems, E, A, S, F;           // F = 2S+1
    int maxw;                            // widest activation vector, multiple of 4
};

// y[o] = act(b[o] + sum_i x[i] W[i][o] (+ Wx[extra][o]))   for o striding over the lanes.
// Weights are packed [i/4][o][i%4] (zero padded) so a lane fetches four weights with one 128-bit
// shared load, and x (shared, 16-byte aligned, zero padded to a multiple of 4) is read as float4
// broadcasts: 2 LDS.128 + 4 FFMA per four inputs.  Entries out..round4(out) of y are zeroed so y
// can feed the next layer's float4 reads.
template <int G>
MZ_DEVINL void linear_layer(const float* __restrict__ W, const float* __restrict__ b, const float* __restrict__ Wx,
                            int in_dense, int out, const float* x, float* y, bool elu, int extra_row) {
    const int lane = LaneGroup<G>::lane();
    const int in4 = (in_dense + 3) >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* W4 = reinterpret_cast<const float4*>(W);
    const int out4 = (out + 3) & ~3;
    for (int o = lane; o < out4; o += G) {
        float r = 0.0f;
        if (o < out) {
            float acc = b[o];
            const float4* w = W4 + o;
#pragma unroll 2
            for (int i = 0; i < in4; ++i) {
                const float4 xv = x4[i];
                const float4 wv = w[i * out];
                acc = fmaf(xv.x, wv.x, acc);
                acc = fmaf(xv.y, wv.y, acc);
                acc = fmaf(xv.z, wv.z, acc);
                acc = fmaf(xv.w, wv.w, acc);
            }
            if (extra_row >= 0) acc += Wx[extra_row * out + o];
            r = elu ? elu1(acc) : acc;
        }
        y[o] = r;
    }
    LaneGroup<G>::sync();
}

// Runs a whole MLP. x must be in shared memory (16-byte aligned, zero padded to a multiple of 4);
// s0/s1 are per-game ping-pong scratch.  For the dynamics net the first layer's input is
// [x | one_hot(action)]: `action` >= 0 selects the one-hot row (models.py:149-155).
// Returns the pointer holding the output (s0, s1 or `final_out` if given).
template <int G>
MZ_DEVINL float* mlp_forward(const MlpDesc& d, const float* blob, const float* x, float* s0, float* s1,
                             float* final_out, int action = -1) {
    const float* cur = x;
    float* dst = s0;
    for (int l = 0; l < d.n; ++l) {
        const bool last = (l == d.n - 1);
        float* y = (last && final_out) ? final_out : dst;
        linear_layer<G>(blob + d.w_off[l], blob + d.b_off[l], d.x_off[l] >= 0 ? blob + d.x_off[l] : nullptr,
                        d.in_dense[l], d.out[l], cur, y, !last, (l == 0) ? action : -1);
        cur = y;
        dst = (y == s0) ? s1 : s0;
    }
    return const_cast<float*>(cur);
}

// K independent MLPs of equal depth evaluated side by side: one instruction stream with K accumulators per
// lane, so the three heads of a recurrent inference (reward on the raw state, policy and value on the rescaled
// state; models.py:157-159,128-131) overlap their shared-memory latencies instead of running back to back.
// Every accumulator sees exactly the operations of linear_layer, in the same order: results are bit-identical.
// bufs: K x 2 ping-pong vectors.  out[k] receives the pointer holding MLP k's output.
template <int G, int K>
MZ_DEVINL void mlp_forward_multi(const MlpDesc* const (&d)[K], const float* blob, const float* const (&x)[K],
                                 float* const (&bufs)[K][2], float* (&out)[K]) {
    const int lane = LaneGroup<G>::lane();
    const float* cur[K];
#pragma unroll
    for (int k = 0; k < K; ++k) cur[k] = x[k];
    const int n_layers = d[0]->n;
    for (int l = 0; l < n_layers; ++l) {
        const bool last = (l == n_layers - 1);
        int in4[K], outk[K], out4[K], max_in4 = 0, max_out4 = 0;
        const float4* W4[K];
        const float* bias[K];
        float* y[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            in4[k] = (d[k]->in_dense[l] + 3) >> 2;
            outk[k] = d[k]->out[l];
            out4[k] = (outk[k] + 3) & ~3;
            W4[k] = reinterpret_cast<const float4*>(blob + d[k]->w_off[l]);
            bias[k] = blob + d[k]->b_off[l];
            y[k] = (l & 1) ? bufs[k][1] : bufs[k][0];
            max_in4 = max(max_in4, in4[k]);
            max_out4 = max(max_out4, out4[k]);
        }
        for (int o = lane; o < max_out4; o += G) {
            float acc[K];
            bool on[K];
#pragma unroll
            for (int k = 0; k < K; ++k) { on[k] = o < outk[k]; acc[k] = on[k] ? bias[k][o] : 0.0f; }
#pragma unroll 2
            for (int i = 0; i < max_in4; ++i) {
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    if (on[k] && i < in4[k]) {
                        const float4 xv = reinterpret_cast<const float4*>(cur[k])[i];
                        const float4 wv = W4[k][i * outk[k] + o];
                        acc[k] = fmaf(xv.x, wv.x, acc[k]);
                        acc[k] = fmaf(xv.y, wv.y, acc[k]);
                        acc[k] = fmaf(xv.z, wv.z, acc[k]);
                        acc[k] = fmaf(xv.w, wv.w, acc[k]);
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < K; ++k)
                if (o < out4[k]) y[k][o] = on[k] ? (last ? acc[k] : elu1(acc[k])) : 0.0f;
        }
        LaneGroup<G>::sync();
#pragma unroll
        for (int k = 0; k < K; ++k) cur[k] = y[k];
    }
#pragma unroll
    for (int k = 0; k < K; ++k) out[k] = const_cast<float*>(cur[k]);
}

// copies n floats from global memory into a zero-padded shared vector
template <int G>
MZ_DEVINL void load_vector(const float* __restrict__ src, float* dst, int n) {
    const int lane = LaneGroup<G>::lane();
    const int n4 = (n + 3) & ~3;
    for (int i = lane; i < n4; i += G) dst[i] = (i < n) ? src[i] : 0.0f;
    LaneGroup<G>::sync();
}

// Per-sample min-max rescale over n values held in shared memory (models.py:138-145,161-168):
// scale = max - min; if (scale < 1e-5) scale += 1e-5; out = (x - min) / scale
template <int G>
MZ_DEVINL void rescale_unit_range(const float* x, float* out, int n) {
    const int lane = LaneGroup<G>::lane();
    float lo = INFINITY, hi = -INFINITY;
    for (int i = lane; i < n; i += G) { lo = fminf(lo, x[i]); hi = fmaxf(hi, x[i]); }
    lo = -group_max_f32<G>(-lo);
    hi = group_max_f32<G>(hi);
    float sc = __fsub_rn(hi, lo);
    if (sc < 1e-5f) sc = __fadd_rn(sc, 1e-5f);
    const int n4 = (n + 3) & ~3;
    for (int i = lane; i < n4; i += G) out[i] = (i < n) ? div_pos_or_zero(__fsub_rn(x[i], lo), sc) : 0.0f;
    LaneGroup<G>::sync();
}

// support_to_scalar (models.py:645-666) of F = 2S+1 logits held in shared memory.
template <int G>
MZ_DEVINL float support_to_scalar_group(const float* logits, int S) {
    const int lane = LaneGroup<G>::lane();
    const int F = 2 * S + 1;
    float m = -INFINITY;
    for (int i = lane; i < F; i += G) m = fmaxf(m, logits[i]);
    m = group_max_f32<G>(m);
    float den = 0.0f, num = 0.0f;
    for (int i = lane; i < F; i += G) {
        const float e = expf(logits[i] - m);
        den += e;
        num = fmaf((float)(i - S), e, num);
    }
    den = group_sum_f32<G>(den);
    num = group_sum_f32<G>(num);
    return inverse_value_transform(__fdiv_rn(num, den));
}

// two support_to_scalar evaluations with interleaved reductions (value and reward heads)
template <int G>
MZ_DEVINL void support_to_scalar_group2(const float* la, const float* lb, int S, float& ra, float& rb) {
    const int lane = LaneGroup<G>::lane();
    const int F = 2 * S + 1;
    const unsigned m = kWarp;
    float ma = -INFINITY, mb = -INFINITY;
    for (int i = lane; i < F; i += G) { ma = fmaxf(ma, la[i]); mb = fmaxf(mb, lb[i]); }
#pragma unroll
    for (int off = G >> 1; off > 0; off >>= 1) {
        ma = fmaxf(ma, __shfl_xor_sync(m, ma, off, G));
        mb = fmaxf(mb, __shfl_xor_sync(m, mb, off, G));
    }
    float da = 0.0f, na = 0.0f, db = 0.0f, nb = 0.0f;
    for (int i = lane; i < F; i += G) {
        const float ea = expf(la[i] - ma), eb = expf(lb[i] - mb);
        da += ea; na = fmaf((float)(i - S), ea, na);
        db += eb; nb = fmaf((float)(i - S), eb, nb);
    }
#pragma unroll
    for (int off = G >> 1; off > 0; off >>= 1) {
        da += __shfl_xor_sync(m, da, off, G); db += __shfl_xor_sync(m, db, off, G);
        na += __shfl_xor_sync(m, na, off, G); nb += __shfl_xor_sync(m, nb, off, G);
    }
    ra = inverse_value_transform(__fdiv_rn(na, da));
    rb = inverse_value_transform(__fdiv_rn(nb, db));
}

// ------------------------------------------------------------------------------------------------------------------
// Fixed-shape recurrent inference (the fused search kernel's per-simulation network call).
//
// The generic code above walks run-time layer descriptors: for CartPole's 8 -> 16 -> {8, 21, 2, 21} networks seven of eight
// instructions it executes are loop control, predicates and address arithmetic.  When the five MLPs have the common shape
//     dynamics  [E | one_hot(A)] -> H -> E          reward / value  E -> H -> F = 2S+1          policy  E -> H -> A
// with compile-time E, H, F, A, everything unrolls: per four inputs one broadcast 128-bit load of x, one 128-bit load of
// the packed weights and four FMAs; the next state, the 2 x F value / reward logits and the policy logit never leave
// registers (no store + barrier + reload between the last layer, the rescale and support_to_scalar).  Every accumulator
// sees the operations of linear_layer / rescale_unit_range / support_to_scalar_group2 in the same order: bit-identical to
// the generic path (tests/test_tree_parity_gpu.py::test_full_size_invariants compares the two on 4096 games).
template <int E_, int H_, int S_, int A_>
struct FcFixedShape {
    static constexpr bool kEnabled = true;
    static constexpr int E = E_, H = H_, S = S_, F = 2 * S_ + 1, A = A_;
    static_assert(E % 4 == 0 && H % 4 == 0, "vector widths");
};
struct FcGenericShape { static constexpr bool kEnabled = false; };

// does the network have the fixed shape SH ?
template <typename SH>
inline bool fc_matches_fixed(const FcNet& n) {
    auto two = [](const MlpDesc& d, int in, int hid, int out) {
        return d.n == 2 && d.in_dense[0] == in && d.out[0] == hid && d.in_dense[1] == hid && d.out[1] == out && d.x_off[1] < 0;
    };
    return n.E == SH::E && n.S == SH::S && n.A == SH::A && two(n.dyn, SH::E, SH::H, SH::E) && n.dyn.x_off[0] >= 0 &&
           two(n.rew, SH::E, SH::H, SH::F) && n.rew.x_off[0] < 0 && two(n.val, SH::E, SH::H, SH::F) && n.val.x_off[0] < 0 &&
           two(n.pol, SH::E, SH::H, SH::A) && n.pol.x_off[0] < 0;
}

// acc = b[o] + sum_i x[i] W[i][o], i ascending, four inputs per step (the accumulation order of linear_layer)
template <int IN>
MZ_DEVINL float dot_packed(const float* __restrict__ W, int out, int o, float bias, const float* x) {
    const float4* W4 = reinterpret_cast<const float4*>(W) + o;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float acc = bias;
#pragma unroll
    for (int i = 0; i < IN / 4; ++i) {
        const float4 xv = x4[i];
        const float4 wv = W4[i * out];
        acc = fmaf(xv.x, wv.x, acc);
        acc = fmaf(xv.y, wv.y, acc);
        acc = fmaf(xv.z, wv.z, acc);
        acc = fmaf(xv.w, wv.w, acc);
    }
    return acc;
}

// One recurrent inference (models.py:147-170, 128-131) of the group's game.  h: parent state (shared, E floats); hn: where
// the rescaled next state goes (shared); s0, s1, sr, sp, sv: shared scratch vectors of >= max(E, H) floats.
// Returns this lane's fp32 prior (lane k <-> action k, 0 in lanes >= A), the scalarised value and reward.
template <int G, typename SH>
MZ_DEVINL void fc_recurrent_fixed(const FcNet& net, const float* blob, const float* h, int action, float* hn,
                                  float* s0, float* s1, float* sr, float* sp, float* sv, float& prior, float& value, float& reward) {
    constexpr int E = SH::E, H = SH::H, F = SH::F, A = SH::A, S = SH::S;
    static_assert(E <= G && A <= G, "one lane per state element / action");
    const int lane = LaneGroup<G>::lane();
    const MlpDesc &dy = net.dyn, &rw = net.rew, &vl = net.val, &pl = net.pol;
    // ---- dynamics layer 1: [h | one_hot(action)] -> H, ELU
#pragma unroll
    for (int o = lane; o < H; o += G) {
        float acc = dot_packed<E>(blob + dy.w_off[0], H, o, blob[dy.b_off[0] + o], h);
        acc += blob[dy.x_off[0] + action * H + o];
        s0[o] = elu1(acc);
    }
    LaneGroup<G>::sync();
    // ---- dynamics layer 2: H -> E (identity); the raw next state stays in a register of lane o and goes to s1 for the reward head
    float raw = 0.0f;
    if (lane < E) {
        raw = dot_packed<H>(blob + dy.w_off[1], E, lane, blob[dy.b_off[1] + lane], s0);
        s1[lane] = raw;
    }
    // ---- min-max rescale over the E values (rescale_unit_range: same extrema, same subtraction and division)
    constexpr int WE = pow2_ceil_c(E);                 // lanes >= E hold the neutral elements: reduce over the first WE lanes
    float lo = lane < E ? raw : INFINITY, hi = lane < E ? raw : -INFINITY;
    lo = -group_max_f32_w<G, WE>(-lo);
    hi = group_max_f32_w<G, WE>(hi);
    float sc = __fsub_rn(hi, lo);
    if (sc < 1e-5f) sc = __fadd_rn(sc, 1e-5f);
    if (lane < E) hn[lane] = div_pos_or_zero(__fsub_rn(raw, lo), sc);
    LaneGroup<G>::sync();
    // ---- first layers of the three heads side by side: reward on the raw state, policy and value on the rescaled one
#pragma unroll
    for (int o = lane; o < H; o += G) {
        const float ar = dot_packed<E>(blob + rw.w_off[0], H, o, blob[rw.b_off[0] + o], s1);
        const float ap = dot_packed<E>(blob + pl.w_off[0], H, o, blob[pl.b_off[0] + o], hn);
        const float av = dot_packed<E>(blob + vl.w_off[0], H, o, blob[vl.b_off[0] + o], hn);
        sr[o] = elu1(ar); sp[o] = elu1(ap); sv[o] = elu1(av);
    }
    LaneGroup<G>::sync();
    // ---- second layers: logits in registers (lane l holds elements l, l + G, ...)
    constexpr int R = (F + G - 1) / G;
    float lr[R], lv[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int o = lane + r * G;
        lr[r] = 0.0f; lv[r] = 0.0f;
        if (o < F) {
            lr[r] = dot_packed<H>(blob + rw.w_off[1], F, o, blob[rw.b_off[1] + o], sr);
            lv[r] = dot_packed<H>(blob + vl.w_off[1], F, o, blob[vl.b_off[1] + o], sv);
        }
    }
    // ---- policy: every lane computes all A logits (the weights and sp are broadcast reads) and evaluates the softmax of
    // tree.cuh::group_softmax_masked over the first W lanes on its own, without shuffles: in each butterfly step entry i
    // combines with entry i ^ off in the operand order lane i used, so lane k's entry k has the bits lane k computed.
    constexpr int W = pow2_ceil_c(A);
    float pe[W], pm[W], ps[W];
#pragma unroll
    for (int i = 0; i < W; ++i) {
        pe[i] = i < A ? dot_packed<H>(blob + pl.w_off[1], A, i, blob[pl.b_off[1] + i], sp) : -INFINITY;
        pm[i] = pe[i];
    }
#pragma unroll
    for (int off = W >> 1; off > 0; off >>= 1) {
        float nx[W];
#pragma unroll
        for (int i = 0; i < W; ++i) nx[i] = fmaxf(pm[i], pm[i ^ off]);
#pragma unroll
        for (int i = 0; i < W; ++i) pm[i] = nx[i];
    }
#pragma unroll
    for (int i = 0; i < W; ++i) { pe[i] = i < A ? expf(pe[i] - pm[i]) : 0.0f; ps[i] = pe[i]; }
#pragma unroll
    for (int off = W >> 1; off > 0; off >>= 1) {
        float nx[W];
#pragma unroll
        for (int i = 0; i < W; ++i) nx[i] = ps[i] + ps[i ^ off];
#pragma unroll
        for (int i = 0; i < W; ++i) ps[i] = nx[i];
    }
    float e_own = 0.0f, s_own = 1.0f;
#pragma unroll
    for (int i = 0; i < A; ++i) if (lane == i) { e_own = pe[i]; s_own = ps[i]; }
    prior = div_pos_or_zero(e_own, s_own);
    // ---- support_to_scalar of value and reward (support_to_scalar_group2 on registers: same maxima, sums and order)
    const unsigned m = kWarp;
    float ma = -INFINITY, mb = -INFINITY;
#pragma unroll
    for (int r = 0; r < R; ++r)
        if (lane + r * G < F) { ma = fmaxf(ma, lv[r]); mb = fmaxf(mb, lr[r]); }
#pragma unroll
    for (int off = G >> 1; off > 0; off >>= 1) {
        ma = fmaxf(ma, __shfl_xor_sync(m, ma, off, G));
        mb = fmaxf(mb, __shfl_xor_sync(m, mb, off, G));
    }
    float da = 0.0f, na = 0.0f, db = 0.0f, nb = 0.0f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int i = lane + r * G;
        if (i < F) {
            const float ea = expf(lv[r] - ma), eb = expf(lr[r] - mb);
            da += ea; na = fmaf((float)(i - S), ea, na);
            db += eb; nb = fmaf((float)(i - S), eb, nb);
        }
    }
#pragma unroll
    for (int off = G >> 1; off > 0; off >>= 1) {
        da += __shfl_xor_sync(m, da, off, G); db += __shfl_xor_sync(m, db, off, G);
        na += __shfl_xor_sync(m, na, off, G); nb += __shfl_xor_sync(m, nb, off, G);
    }
    // every lane holds the four sums: the lower half of the group scalarises the value, the upper half the reward - one
    // division and one inverse transform per instruction stream instead of two - and two shuffles share the results
    const bool upper = lane >= G / 2;
    const float tr = inverse_value_transform(__fdiv_rn(upper ? nb : na, upper ? db : da));
    value = __shfl_sync(m, tr, 0, G);
    reward = __shfl_sync(m, tr, G / 2, G);
    LaneGroup<G>::sync();                              // sr / sp / sv / s0 / s1 are free again
}

}  // namespace mz
