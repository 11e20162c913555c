// Step-wise tree kernel for wide action spaces, 32 < |A| <= 256 (games/gomoku.py: 121 actions on 11 x 11, 225 on 15 x 15).
//
// Same arithmetic, same operation order and same pool layout as tree_kernels.cu / tree.cuh (select_child / ucb_score
// self_play.py:363-404, Node.expand :451-465, add_exploration_noise :467-476, backpropagate :406-430); the only change is
// the mapping of children to lanes: one WARP owns a game and lane l scores the children l, l + 32, ..., l + 32 (kJ - 1),
// so a level costs up to kJ rounds of the per-child work and the tie list is kJ ballot words read in ascending action
// order.  kJ is a template parameter, 4 for |A| <= 128 and 8 for |A| <= 256, and nothing but trip counts depends on it.
// The backup does not depend on |A| and is tree.cuh's.  Kept apart from the narrow kernel on purpose: the
// per-simulation kernel of the BASELINE configs (|A| <= 9) keeps its register budget and its tested code path.
#include <stdlib.h>

#include "kernels.h"
#include "launch.h"
#include "pipeline.h"
#include "tree.cuh"

namespace mz {

namespace {

constexpr int kLegalWords = MZ_MAX_ACTIONS / 32;      // words of a game's legal mask in the pool, whatever kJ reads of them
using LG = LaneGroup<32>;

// lowest set bit position across the words in ascending action order, or the n-th (0-based) set bit
template <int kJ>
MZ_DEVINL int nth_action(const unsigned (&w)[kJ], int n) {
#pragma unroll
    for (int j = 0; j < kJ; ++j) {
        const int c = __popc(w[j]);
        if (n < c) return 32 * j + nth_set_bit(w[j], n);
        n -= c;
    }
    return 0;
}

}  // namespace

// kJ: children per lane.  With eight, the register allocator's default target leaves five of the legal-mask words in
// local memory; one resident CTA per SM as the stated minimum lifts that target (189 registers, no spills) and leaves
// the kJ = 4 instantiation, which states none, as it was (128 registers).
template <int kJ>
__global__ void __launch_bounds__(128, kJ > 4 ? 1 : 0) tree_step_wide_kernel(const __grid_constant__ TreeStepArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int local = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (local >= a.n) return;
    const int g = a.g0 + local;
    const int lane = threadIdx.x & 31;
    const int N = a.N, A = a.A;
    const size_t slots = (size_t)(N + 1) * A;
    const NodePool& p = a.pool;

    TreeConst c;
    c.A = A; c.N = N; c.P = a.P; c.discount = a.discount; c.noise_frac = a.noise_frac; c.noise_alpha = a.noise_alpha; c.seed = a.seed;
    c.pbc = a.pbc; c.sqrtn = a.sqrtn; c.ucb = a.ucb;

    GameTree t;
    t.visit = p.visit + g * slots;
    t.vsum = p.vsum + g * slots;
    t.mval = p.mval + g * slots;
    t.reward = p.reward + g * slots;
    t.prior = p.prior + g * slots;
    t.expansion = p.expansion + g * slots;
    t.root_prior = p.root_prior + (size_t)g * A;
    t.path = p.path + (size_t)g * (N + 2);
    t.path_reward = p.path_reward + (size_t)g * (N + 2);
    unsigned legal[kJ];
    int max_depth = 0;
    const int64_t game_id = a.game_id ? a.game_id[g] : (int64_t)g;
    const int move = a.move_index ? a.move_index[g] : 0;

    // fp32 softmax over the children `ok` marks (self_play.py:460-462): this lane's priors for its kJ children
    auto softmax = [&](const float (&logit)[kJ], const bool (&ok)[kJ], float (&prior)[kJ]) {
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < kJ; ++j) if (ok[j]) m = fmaxf(m, logit[j]);
        m = group_max_f32<32>(m);
        float e[kJ], s = 0.0f;
#pragma unroll
        for (int j = 0; j < kJ; ++j) { e[j] = ok[j] ? expf(logit[j] - m) : 0.0f; s += e[j]; }
        s = group_sum_f32<32>(s);
#pragma unroll
        for (int j = 0; j < kJ; ++j) prior[j] = div_pos_or_zero(e[j], s);
    };

    if (a.do_root == 1) {
        float logit[kJ], prior[kJ];
        bool ok[kJ];
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
            const int k = lane + 32 * j;
            const bool is_legal = k < A && (a.legal_mask == nullptr || a.legal_mask[(size_t)g * A + k]);
            legal[j] = __ballot_sync(0xffffffffu, is_legal);
            ok[j] = is_legal;
            logit[j] = k < A ? a.net_policy[(size_t)g * a.policy_stride + k] : 0.0f;
        }
        if (a.policy_is_prior) {
#pragma unroll
            for (int j = 0; j < kJ; ++j) prior[j] = logit[j];
        } else {
            softmax(logit, ok, prior);
        }
        const float root_reward = a.net_reward ? a.net_reward[(size_t)g * a.value_stride] : inverse_value_transform(0.0f);
        // Dirichlet noise: given by action id, or drawn here (normalised Gamma(alpha) draws over the legal actions)
        double nz[kJ];
        const bool have_noise = a.add_noise != 0;
        if (a.add_noise && !a.noise) {
            double sum = 0.0;
#pragma unroll
            for (int j = 0; j < kJ; ++j) { nz[j] = ok[j] ? philox_gamma(a.seed, game_id, move, lane + 32 * j, a.noise_alpha) : 0.0; sum += nz[j]; }
            for (int off = 16; off > 0; off >>= 1) sum += shfl_xor_f64(0xffffffffu, sum, off, 32);
#pragma unroll
            for (int j = 0; j < kJ; ++j) nz[j] = nz[j] / sum;
        } else {
#pragma unroll
            for (int j = 0; j < kJ; ++j) nz[j] = (a.add_noise && ok[j]) ? a.noise[(size_t)g * A + lane + 32 * j] : 0.0;
        }
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
            const int k = lane + 32 * j;
            if (k >= A) continue;
            if (a.trace.root_priors_raw) a.trace.root_priors_raw[(size_t)g * A + k] = ok[j] ? prior[j] : 0.0f;
            if (a.trace.noise) a.trace.noise[(size_t)g * A + k] = nz[j];
            double pr = (double)prior[j];
            if (ok[j] && have_noise)
                pr = __dadd_rn(__dmul_rn(pr, __dsub_rn(1.0, c.noise_frac)), __dmul_rn(nz[j], c.noise_frac));      // self_play.py:476
            t.root_prior[k] = ok[j] ? pr : 0.0;
            t.visit[k] = 0;
            t.vsum[k] = 0.0;
            t.reward[k] = 0.0f;
            t.prior[k] = ok[j] ? prior[j] : 0.0f;
            t.expansion[k] = -1;
        }
        if (a.trace.root_reward && lane == 0) a.trace.root_reward[g] = root_reward;
        if (lane == 0 && a.root_predicted_value) a.root_predicted_value[g] = a.net_value[(size_t)g * a.value_stride];
        t.root_visit = 0; t.root_vsum = 0.0; t.root_reward = root_reward;
        t.lo = INFINITY; t.hi = -INFINITY; t.n_expanded = 1; t.ties = 0;
        __syncwarp();
    } else {
#pragma unroll
        for (int j = 0; j < kJ; ++j) legal[j] = p.legal[(size_t)g * kLegalWords + j];
        t.root_visit = p.root_visit[g];
        t.root_vsum = p.root_vsum[g];
        t.root_reward = p.root_reward[g];
        t.lo = p.range[2 * g];
        t.hi = p.range[2 * g + 1];
        t.n_expanded = p.n_expanded[g];
        t.ties = p.ties[g];
        max_depth = p.max_depth[g];
    }

    if (a.do_update) {
        Leaf leaf;
        leaf.depth = p.leaf_depth[g];
        leaf.parent_exp = p.leaf_parent[g];
        leaf.action = p.leaf_action[g];
        leaf.slot = p.leaf_slot[g];
        const float value = a.net_value[(size_t)g * a.value_stride];
        const float reward = a.net_reward[(size_t)g * a.value_stride];
        float logit[kJ], prior[kJ];
        bool ok[kJ];
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
            const int k = lane + 32 * j;
            ok[j] = k < A;
            logit[j] = ok[j] ? a.net_policy[(size_t)g * a.policy_stride + k] : 0.0f;
        }
        if (a.policy_is_prior) {
#pragma unroll
            for (int j = 0; j < kJ; ++j) prior[j] = logit[j];
        } else {
            softmax(logit, ok, prior);
        }
        if (a.trace.depth) {
            const int sim = a.sim - 1;
            const size_t ti = (size_t)g * N + sim;
            if (lane == 0) { a.trace.depth[ti] = leaf.depth; a.trace.value[ti] = value; a.trace.reward[ti] = reward; }
#pragma unroll
            for (int j = 0; j < kJ; ++j) if (ok[j]) a.trace.priors[ti * A + lane + 32 * j] = prior[j];
            for (int d = lane; d < leaf.depth && d < a.trace.max_depth; d += 32)
                a.trace.actions[ti * a.trace.max_depth + d] = (uint8_t)(t.path[d + 1] % A);
        }
        // Node.expand (self_play.py:451-465): the leaf becomes expansion e, its |A| children are created eagerly
        const int e = t.n_expanded;
        if (lane == 0) {
            t.expansion[leaf.slot] = e;
            t.reward[leaf.slot] = reward;
            t.path_reward[leaf.depth] = reward;
        }
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
            if (!ok[j]) continue;
            const int s = e * A + lane + 32 * j;
            t.visit[s] = 0;
            t.vsum[s] = 0.0;
            t.reward[s] = 0.0f;
            t.prior[s] = prior[j];
            t.expansion[s] = -1;
        }
        t.n_expanded = e + 1;
        __syncwarp();
        tree_backup<32>(c, t, leaf, value);
        max_depth = max(max_depth, leaf.depth);
    }

    if (a.do_select) {
        const int first_index = a.first_index ? a.first_index[g] : -1;
        int e = 0, n_parent = t.root_visit, depth = 0;
        Leaf leaf;
        if (lane == 0) { t.path[0] = -1; t.path_reward[0] = t.root_reward; }
        while (true) {
            const int base = e * A;
            double score[kJ];
            int nc[kJ], cexp[kJ];
            float rew[kJ];
            bool valid[kJ];
            double local_best = -INFINITY;
#pragma unroll
            for (int j = 0; j < kJ; ++j) {
                const int k = lane + 32 * j;
                valid[j] = k < A && (e != 0 || ((legal[j] >> lane) & 1u));
                score[j] = -INFINITY; nc[j] = 0; cexp[j] = -1; rew[j] = 0.0f;
                if (valid[j]) {
                    nc[j] = t.visit[base + k];
                    cexp[j] = t.expansion[base + k];
                    const double pr = (e == 0) ? t.root_prior[k] : (double)t.prior[base + k];
                    // pb_c = (log(...) + init) * (sqrt(n_p) / (n_c + 1))     self_play.py:384-390
                    double pbc;
                    if (c.ucb) pbc = __ldg(c.ucb + n_parent * (c.N + 2) + nc[j]);
                    else pbc = __dmul_rn(c.pbc[n_parent], __ddiv_rn(c.sqrtn[n_parent], (double)(nc[j] + 1)));
                    double s = __dmul_rn(pbc, pr);
                    if (nc[j] > 0) {
                        rew[j] = t.reward[base + k];
                        s = __dadd_rn(s, value_range_normalize(t.mval[base + k], t.lo, t.hi));
                    } else {
                        s = __dadd_rn(s, 0.0);
                    }
                    score[j] = s;
                    local_best = fmax(local_best, s);
                }
            }
            const double best = group_max_f64<32>(local_best, 32);
            unsigned tied[kJ];
            int n_tied = 0;
#pragma unroll
            for (int j = 0; j < kJ; ++j) { tied[j] = __ballot_sync(0xffffffffu, valid[j] && score[j] == best); n_tied += __popc(tied[j]); }
            int pick;
            if (n_tied <= 1) {
                pick = nth_action(tied, 0);
            } else {
                int idx;
                if (a.sim == 0 && depth == 0 && first_index >= 0) {
                    idx = first_index < n_tied ? first_index : n_tied - 1;
                } else {
                    idx = philox_tie_index(c.seed, game_id, move, a.sim, depth, n_tied);
                    if (!(a.sim == 0 && depth == 0)) t.ties += 1;
                }
                pick = nth_action(tied, idx);
            }
            const int pj = pick >> 5, pl = pick & 31;
            int sel_exp = -1, sel_nc = 0;
            float sel_rew = 0.0f;
#pragma unroll
            for (int j = 0; j < kJ; ++j) if (j == pj) { sel_exp = cexp[j]; sel_nc = nc[j]; sel_rew = rew[j]; }
            const int child_exp = __shfl_sync(0xffffffffu, sel_exp, pl);
            const int child_visits = __shfl_sync(0xffffffffu, sel_nc, pl);
            const int slot = base + pick;
            depth += 1;
            if (lane == pl) { t.path[depth] = slot; t.path_reward[depth] = sel_rew; }
            if (child_exp < 0) {
                leaf.depth = depth; leaf.parent_exp = e; leaf.action = pick; leaf.slot = slot;
                break;
            }
            n_parent = child_visits;
            e = child_exp;
        }
        __syncwarp();
        if (lane == 0) {
            p.leaf_depth[g] = leaf.depth;
            p.leaf_parent[g] = leaf.parent_exp;
            p.leaf_action[g] = leaf.action;
            p.leaf_slot[g] = leaf.slot;
        }
    }

    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < kJ; ++j) p.legal[(size_t)g * kLegalWords + j] = legal[j];
        p.root_visit[g] = t.root_visit;
        p.root_vsum[g] = t.root_vsum;
        p.root_reward[g] = t.root_reward;
        p.range[2 * g] = t.lo;
        p.range[2 * g + 1] = t.hi;
        p.n_expanded[g] = t.n_expanded;
        p.ties[g] = t.ties;
        p.max_depth[g] = max_depth;
    }

    if (a.do_final) {
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
            const int k = lane + 32 * j;
            if (k >= A) continue;
            const bool ok = (legal[j] >> lane) & 1u;
            if (a.visit_counts) a.visit_counts[(size_t)g * A + k] = ok ? t.visit[k] : 0;
            if (a.root_priors) a.root_priors[(size_t)g * A + k] = t.root_prior[k];
        }
        if (lane == 0) {
            if (a.root_value) a.root_value[g] = (t.root_visit == 0) ? 0.0 : __ddiv_rn(t.root_vsum, (double)t.root_visit);
            if (a.max_tree_depth) a.max_tree_depth[g] = max_depth;
            if (a.tie_count) a.tie_count[g] = t.ties;
            if (a.value_range) { a.value_range[2 * g] = t.lo; a.value_range[2 * g + 1] = t.hi; }
        }
    }
}

cudaError_t launch_tree_step_wide(const TreeStepArgs& a, cudaStream_t stream) {
    const int grid = (a.n * 32 + 127) / 128;
    cudaError_t e = a.A <= 128 ? launch_chained(tree_step_wide_kernel<4>, dim3(grid), dim3(128), 0, stream, a)
                               : launch_chained(tree_step_wide_kernel<8>, dim3(grid), dim3(128), 0, stream, a);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace mz
