// One game's share of a step-wise tree launch (tree_kernels.cu) as a device function, so that the per-simulation kernel
// and the fused small-network search kernel (small_search.cu) execute the SAME code:
//   [root expansion] -> [expand + backup of the previous simulation's leaf] -> [selection of the next leaf] -> [read-out]
// A group of G >= |A| lanes owns game g (global index into the node pool).  `sim` is the simulation selected by this
// step (do_select); do_update handles sim - 1.  own = false: the group has no game of its own and replays game g, which
// belongs to another group of its warp, without storing anything (the warp's collectives need every group, see LaneGroup).
#pragma once
#include "kernels.h"
#include "pipeline.h"
#include "tree.cuh"

namespace mz {

template <int G, bool kLatency>
MZ_DEVINL void tree_step_game(const TreeStepArgs& a, int g, bool own, int sim, int do_root, int do_update, int do_select,
                               int do_final) {
    const int lane = LaneGroup<G>::lane();
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
    t.own = own;
    int max_depth = 0;

    if (do_root == 1) {
        unsigned legal = 0;
        for (int k = 0; k < A; ++k)
            legal |= (a.legal_mask == nullptr || a.legal_mask[(size_t)g * A + k]) ? (1u << k) : 0u;
        t.legal = legal;
        const bool ok = lane < A && ((legal >> lane) & 1u);
        float prior;
        if (a.policy_is_prior) prior = (lane < A) ? a.net_policy[(size_t)g * a.policy_stride + lane] : 0.0f;
        else prior = group_softmax_masked<G>((lane < A) ? a.net_policy[(size_t)g * a.policy_stride + lane] : 0.0f, ok);
        const float root_reward = a.net_reward ? a.net_reward[(size_t)g * a.value_stride] : inverse_value_transform(0.0f);
        if (a.trace.root_priors_raw && lane < A && own) a.trace.root_priors_raw[(size_t)g * A + lane] = ok ? prior : 0.0f;
        if (a.trace.root_reward && lane == 0 && own) a.trace.root_reward[g] = root_reward;
        tree_init_root<G>(c, t, prior, root_reward, (a.add_noise && a.noise) ? a.noise + (size_t)g * A : nullptr,
                          a.add_noise && !a.noise, a.game_id ? a.game_id[g] : (int64_t)g, a.move_index ? a.move_index[g] : 0,
                          a.trace.noise ? a.trace.noise + (size_t)g * A : nullptr);
        if (lane == 0 && own && a.root_predicted_value) a.root_predicted_value[g] = a.net_value[(size_t)g * a.value_stride];
    } else {
        t.legal = p.legal[g];
        t.root_visit = p.root_visit[g];
        t.root_vsum = p.root_vsum[g];
        t.root_reward = p.root_reward[g];
        t.lo = p.range[2 * g];
        t.hi = p.range[2 * g + 1];
        t.n_expanded = p.n_expanded[g];
        t.ties = p.ties[g];
        max_depth = p.max_depth[g];
    }

    if (do_update) {
        Leaf leaf;
        leaf.depth = p.leaf_depth[g];
        leaf.parent_exp = p.leaf_parent[g];
        leaf.action = p.leaf_action[g];
        leaf.slot = p.leaf_slot[g];
        const float value = a.net_value[(size_t)g * a.value_stride];
        const float reward = a.net_reward[(size_t)g * a.value_stride];
        float prior;
        if (a.policy_is_prior) prior = (lane < A) ? a.net_policy[(size_t)g * a.policy_stride + lane] : 0.0f;
        else prior = group_softmax_masked<G>((lane < A) ? a.net_policy[(size_t)g * a.policy_stride + lane] : 0.0f, lane < A);
        if (a.trace.depth && own) {
            const size_t ti = (size_t)g * N + (sim - 1);
            if (lane == 0) { a.trace.depth[ti] = leaf.depth; a.trace.value[ti] = value; a.trace.reward[ti] = reward; }
            if (lane < A) a.trace.priors[ti * A + lane] = prior;
            for (int j = lane; j < leaf.depth && j < a.trace.max_depth; j += G)
                a.trace.actions[ti * a.trace.max_depth + j] = (uint8_t)(t.path[j + 1] % A);
        }
        tree_expand<G>(c, t, leaf, reward, prior);
        tree_backup<G>(c, t, leaf, value);
        max_depth = max(max_depth, leaf.depth);
    }

    if (do_select) {
        const int64_t game_id = a.game_id ? a.game_id[g] : (int64_t)g;
        const int move = a.move_index ? a.move_index[g] : 0;
        const int first_index = a.first_index ? a.first_index[g] : -1;
        const Leaf leaf = tree_select<G, kLatency>(c, t, sim, game_id, move, first_index);
        if (lane == 0 && own) {
            p.leaf_depth[g] = leaf.depth;
            p.leaf_parent[g] = leaf.parent_exp;
            p.leaf_action[g] = leaf.action;
            p.leaf_slot[g] = leaf.slot;
        }
    }

    if (lane == 0 && own) {
        p.legal[g] = t.legal;
        p.root_visit[g] = t.root_visit;
        p.root_vsum[g] = t.root_vsum;
        p.root_reward[g] = t.root_reward;
        p.range[2 * g] = t.lo;
        p.range[2 * g + 1] = t.hi;
        p.n_expanded[g] = t.n_expanded;
        p.ties[g] = t.ties;
        p.max_depth[g] = max_depth;
    }

    if (do_final && own) {
        if (lane < A) {
            const bool ok = (t.legal >> lane) & 1u;
            if (a.visit_counts) a.visit_counts[(size_t)g * A + lane] = ok ? t.visit[lane] : 0;
            if (a.root_priors) a.root_priors[(size_t)g * A + lane] = t.root_prior[lane];
        }
        if (lane == 0) {
            if (a.root_value) a.root_value[g] = (t.root_visit == 0) ? 0.0 : __ddiv_rn(t.root_vsum, (double)t.root_visit);
            if (a.max_tree_depth) a.max_tree_depth[g] = max_depth;
            if (a.tie_count) a.tie_count[g] = t.ties;
            if (a.value_range) { a.value_range[2 * g] = t.lo; a.value_range[2 * g + 1] = t.hi; }
        }
    }
}

}  // namespace mz
