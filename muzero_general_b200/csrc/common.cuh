// Shared device helpers: lane groups, reductions, Philox4x32-10, fp32 scalarisation.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define MZ_DEVINL __device__ __forceinline__

#include "philox.cuh"

namespace mz {

// ------------------------------------------------------------------------------------------
// Lane groups: a warp is split into 32/G groups of G consecutive lanes; one game per group.
//
// Every group of a warp calls every collective, the same number of times, so that each one takes the constant full mask
// (kWarp) and the segment width G keeps the groups' data apart.  A mask that depends on the lane (0xffff << 16 for the
// upper group of G = 16) makes nvcc guard each collective region with a run-time convergence check (MATCH.ANY, REDUX.OR,
// a divergent-branch fallback); the full mask needs none.  Hence: a loop that contains a collective runs to the largest
// trip count of the warp's groups (the others predicate their updates off), and a persistent loop over games iterates
// while the warp still has a game - a group without one runs on a clamped index and stores nothing.
// ------------------------------------------------------------------------------------------
constexpr unsigned kWarp = 0xffffffffu;

template <int G>
struct LaneGroup {
    static_assert(G == 4 || G == 8 || G == 16 || G == 32, "group width");
    MZ_DEVINL static unsigned lane() { return threadIdx.x & (G - 1); }
    MZ_DEVINL static unsigned base() { return (threadIdx.x & 31u) & ~(unsigned)(G - 1); }
    MZ_DEVINL static void sync() { __syncwarp(kWarp); }
    // ballot restricted to the group, bit i = lane i of the group
    MZ_DEVINL static unsigned ballot(bool p) {
        unsigned b = __ballot_sync(kWarp, p);
        if constexpr (G == 32) return b;
        else return (b >> base()) & ((1u << G) - 1u);
    }
    template <typename T>
    MZ_DEVINL static T bcast(T v, int src) { return __shfl_sync(kWarp, v, src, G); }
    // true in every lane while any group of the warp passes p (the trip-count test of a loop that contains collectives)
    MZ_DEVINL static bool warp_any(bool p) { return __any_sync(kWarp, p); }
    // Waits until all 32 lanes of the warp are converged here (WARPSYNC.ALL).  Where ptxas cannot prove the warp converged
    // at a collective - after a loop whose trip count depends on threadIdx, such as the persistent loop over games - it
    // wraps the collective in a run-time divergence test (BRA.DIV) with an out-of-line WARPSYNC.COLLECTIVE / ENDCOLLECTIVE
    // fallback, and since that fallback may rejoin diverged, every later collective gets one too.  A warp-wide reduction
    // needs a converged warp and its WARPSYNC.ALL re-establishes the proof: placed in front of a loop whose every path
    // ends converged, it leaves the loop's collectives without any test.  (An asm volatile, so that the unused result
    // does not let the compiler drop it.)
    MZ_DEVINL static void converge() {
        unsigned r;
        asm volatile("redux.sync.or.b32 %0, %1, 0xffffffff;" : "=r"(r) : "r"(0u));
    }
};

MZ_DEVINL double shfl_xor_f64(unsigned mask, double v, int off, int width) {
    int lo = __double2loint(v), hi = __double2hiint(v);
    lo = __shfl_xor_sync(mask, lo, off, width);
    hi = __shfl_xor_sync(mask, hi, off, width);
    return __hiloint2double(hi, lo);
}
MZ_DEVINL double shfl_f64(unsigned mask, double v, int src, int width) {
    int lo = __double2loint(v), hi = __double2hiint(v);
    lo = __shfl_sync(mask, lo, src, width);
    hi = __shfl_sync(mask, hi, src, width);
    return __hiloint2double(hi, lo);
}

// smallest power of two >= n (n >= 1)
// d / sc (IEEE round-to-nearest) for sc > 0.  A zero numerator - every channel minimum, every ReLU zero - sends
// div.rn.f32 down its out-of-line slow path (FCHK rejects zero / denormal operands) and the whole warp waits for it;
// 0 / sc is +0 anyway, so divide a harmless 1.0 instead and select.
MZ_DEVINL float div_pos_or_zero(float d, float sc) {
    const float q = __fdiv_rn(d == 0.0f ? 1.0f : d, sc);
    return d == 0.0f ? 0.0f : q;
}

// hint: bring the line holding *p into L1 (no register, no dependency)
MZ_DEVINL void prefetch_l1(const void* p) { asm volatile("prefetch.L1 [%0];" ::"l"(p)); }

MZ_DEVINL int pow2_ceil(int n) { return n <= 1 ? 1 : 1 << (32 - __clz(n - 1)); }

// Exact max / min (no rounding involved), NaN-free inputs assumed.  `width` must be the same in every group of the warp.
template <int G>
MZ_DEVINL double group_max_f64(double v, int width) {
    for (int off = width >> 1; off > 0; off >>= 1) v = fmax(v, shfl_xor_f64(kWarp, v, off, G));
    return v;
}
template <int G>
MZ_DEVINL double group_min_f64(double v, int width) {
    for (int off = width >> 1; off > 0; off >>= 1) v = fmin(v, shfl_xor_f64(kWarp, v, off, G));
    return v;
}
template <int G>
MZ_DEVINL float group_max_f32(float v) {
#pragma unroll
    for (int off = G >> 1; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kWarp, v, off, G));
    return v;
}
// The same reductions over the first W lanes of the group only (W a power of two <= G): valid in lanes < W.  With the lanes
// >= W holding the neutral element the full-width reduction returns the same bits (max is exact, x + 0 is exact): these
// just skip the steps that cannot change the result.
constexpr int pow2_ceil_c(int n) { return n <= 1 ? 1 : 2 * pow2_ceil_c((n + 1) / 2); }
template <int G, int W>
MZ_DEVINL float group_max_f32_w(float v) {
#pragma unroll
    for (int off = W >> 1; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kWarp, v, off, G));
    return v;
}
template <int G, int W>
MZ_DEVINL float group_sum_f32_w(float v) {
#pragma unroll
    for (int off = W >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(kWarp, v, off, G);
    return v;
}
template <int G>
MZ_DEVINL float group_sum_f32(float v) {
#pragma unroll
    for (int off = G >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(kWarp, v, off, G);
    return v;
}

// ------------------------------------------------------------------------------------------
// Philox4x32-10 draws (philox.cuh)
// ------------------------------------------------------------------------------------------
// index in [0, n) for an exact UCB tie at (game, move, sim, depth)
MZ_DEVINL int philox_tie_index(uint64_t seed, int64_t game, int move, int sim, int depth, int n) {
    const Philox4 r = philox4x32_10((uint32_t)game, (uint32_t)move, (uint32_t)sim, (uint32_t)depth,
                                    (uint32_t)seed, (uint32_t)(seed >> 32) ^ kTagTie);
    return (int)__umulhi(r.x, (uint32_t)n);
}

// Gamma(alpha, 1) sample for lane-private use (Marsaglia & Tsang 2000, with the alpha < 1 boost
// gamma(alpha) = gamma(alpha+1) * U^(1/alpha)); uniforms from Philox keyed (game, move, lane, draw).
// Used to draw the root Dirichlet noise on the device (self_play.py:473) when the host passes none.
static __device__ __noinline__ double philox_gamma(uint64_t seed, int64_t game, int move, int lane, double alpha) {
    const double a = alpha < 1.0 ? alpha + 1.0 : alpha;
    const double d = a - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
    const double k2 = 1.0 / 4294967296.0;
    double out = d;
    for (int it = 0; it < 64; ++it) {
        const Philox4 r = philox4x32_10((uint32_t)game, (uint32_t)move, (uint32_t)lane, (uint32_t)it,
                                        (uint32_t)seed, (uint32_t)(seed >> 32) ^ kTagNoise);
        const double u1 = ((double)r.x + 0.5) * k2, u2 = ((double)r.y + 0.5) * k2, u3 = ((double)r.z + 0.5) * k2;
        const double x = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);          // Box-Muller
        const double t = 1.0 + c * x;
        if (t <= 0.0) continue;
        const double v = t * t * t;
        if (log(u3) < 0.5 * x * x + d - d * v + d * log(v)) { out = d * v; break; }
    }
    if (alpha < 1.0) {
        const Philox4 r = philox4x32_10((uint32_t)game, (uint32_t)move, (uint32_t)lane, 0xFFFFu,
                                        (uint32_t)seed, (uint32_t)(seed >> 32) ^ kTagNoise);
        out *= pow(((double)r.x + 0.5) * k2, 1.0 / alpha);
    }
    return out;
}

// ------------------------------------------------------------------------------------------
// fp32 helpers written with explicit rounding so -fmad cannot change them.
// ------------------------------------------------------------------------------------------
// models.py:661-665 applied to x = sum_k k * softmax(logits)_k
MZ_DEVINL float inverse_value_transform(float x) {
    const float eps = 0.001f;
    const float ax = fabsf(x);
    float t = __fadd_rn(__fadd_rn(ax, 1.0f), eps);          // |x| + 1 + 0.001
    t = __fadd_rn(1.0f, __fmul_rn(4.0f * eps, t));          // 1 + 4*0.001*(...)
    t = __fsub_rn(__fsqrt_rn(t), 1.0f);                     // sqrt(...) - 1
    t = __fdiv_rn(t, 2.0f * eps);                           // / (2*0.001)
    t = __fsub_rn(__fmul_rn(t, t), 1.0f);                   // **2 - 1
    const float sgn = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f);   // torch.sign
    return __fmul_rn(sgn, t);
}

MZ_DEVINL float elu1(float x) { return x > 0.0f ? x : (expf(x) - 1.0f); }

}  // namespace mz
