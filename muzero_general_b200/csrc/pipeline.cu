// Orchestration of the step-wise search: N+1 tree launches with the batched network call
// in between (MCTS.run, self_play.py:260-361, for a whole batch of games in lockstep).
#include "pipeline.h"
#include "ktimer.h"

namespace mz {

int run_stepwise_search(const MzNetDesc& net, const MzSearchDesc& search, int pool_n, const NodePool& pool, const double* d_pbc,
                        const double* d_sqrt, const double* d_ucb, const FcNet& fc, const float* d_fc_blob, ResNetDevice* res,
                        const SearchCall& call, int fc_group, int sm_count, size_t smem_cap, cudaStream_t stream, int64_t* launches,
                        std::string* err) {
    // N = simulations of this call; NP = the layout size of the pool / tables (N + extra_expansions)
    const int n = call.n, N = search.num_simulations, NP = pool_n, A = net.action_space;
    const bool teacher = call.teacher.root_value != nullptr;
    const int K0 = call.continue_from;                 // expansions already in the pool (MZ_FLAG_CONTINUE), else 0
    auto cuda_fail = [&](const char* what, cudaError_t e) {
        *err = std::string(what) + ": " + cudaGetErrorString(e);
        return MZ_ECUDA;
    };
    auto infer = [&](const InferCall& c) -> int {
        if (net.kind == MZ_NET_FC) {
            kt_begin(KT_OTHER, stream);
            cudaError_t e = launch_fc_inference_pool(fc, d_fc_blob, c, fc_group, sm_count, smem_cap, stream);
            kt_end(stream);
            if (e != cudaSuccess) return cuda_fail("fc_inference", e);
            *launches += 1;
            return MZ_OK;
        }
        return resnet_inference(res, c, stream, launches, err);
    };

    const bool run_root = call.phases == kPhaseAll || (call.phases & kPhaseRoot);
    const bool run_sims = call.phases == kPhaseAll || (call.phases & kPhaseSims);
    TreeStepArgs a{};
    a.g0 = call.g0;
    a.n = n; a.N = NP; a.A = A; a.P = search.num_players;
    a.discount = search.discount; a.noise_frac = search.root_exploration_fraction; a.noise_alpha = search.root_dirichlet_alpha; a.seed = search.seed;
    a.pbc = d_pbc; a.sqrtn = d_sqrt; a.ucb = d_ucb; a.pool = pool;
    a.legal_mask = call.legal_mask; a.noise = call.noise; a.add_noise = call.add_noise;
    a.first_index = call.first_index; a.game_id = call.game_id; a.move_index = call.move_index;
    a.visit_counts = call.visit_counts; a.root_value = call.root_value; a.root_predicted_value = call.root_predicted_value;
    a.max_tree_depth = call.max_tree_depth; a.tie_count = call.tie_count; a.root_priors = call.root_priors;
    a.value_range = call.value_range; a.trace = call.trace;

    // ---- root
    cudaError_t e = cudaSuccess;
    if (run_root) {
    if (K0 > 0) {
        a.net_value = pool.net_value; a.net_reward = nullptr; a.net_policy = pool.net_policy;     // unused by do_root == 2
        a.value_stride = 1; a.policy_stride = A; a.policy_is_prior = 0;
    } else if (teacher) {
        a.net_value = call.teacher.root_value; a.net_reward = call.teacher.root_reward; a.net_policy = call.teacher.root_priors;
        a.value_stride = 1; a.policy_stride = A; a.policy_is_prior = 1;
    } else {
        InferCall c{};
        c.n = n; c.g0 = call.g0; c.recurrent = 0; c.in = call.obs;
        c.pool_hidden = pool.hidden; c.pool_stride = NP + 1; c.out_slot = 0;
        c.value = pool.net_value; c.policy_logits = pool.net_policy;
        int rc = infer(c);
        if (rc) return rc;
        a.net_value = pool.net_value; a.net_reward = nullptr; a.net_policy = pool.net_policy;
        a.value_stride = 1; a.policy_stride = A; a.policy_is_prior = 0;
    }
    a.sim = 0; a.do_root = K0 > 0 ? 0 : 1; a.do_update = 0; a.do_select = N > 0; a.do_final = N == 0;
    kt_begin(KT_TREE, stream);
    if (K0 > 0) { e = launch_tree_adopt_root(a, stream); *launches += 1; }
    if (e == cudaSuccess) e = launch_tree_step(a, stream);
    kt_end(stream);
    if (e != cudaSuccess) return cuda_fail("tree_step(root)", e);
    *launches += 1;
    }
    if (!run_sims) return MZ_OK;

    // ---- simulations
    if (!teacher && net.kind == MZ_NET_RESNET && K0 == 0 && N > 0 && !call.trace.depth) {
        // small residual networks: ONE launch runs every simulation of every game (small_search.cu)
        InferCall c{};
        c.n = n; c.g0 = call.g0; c.recurrent = 1; c.action = pool.leaf_action; c.gather_parent = pool.leaf_parent;
        c.pool_hidden = pool.hidden; c.pool_stride = NP + 1; c.out_slot = 1;
        c.value = pool.net_value; c.reward = pool.net_reward; c.policy_logits = pool.net_policy;
        a.net_value = pool.net_value; a.net_reward = pool.net_reward; a.net_policy = pool.net_policy;
        a.value_stride = 1; a.policy_stride = A; a.policy_is_prior = 0;
        if (resnet_small_search_supported(res, c, a, N)) return resnet_small_search(res, c, a, N, stream, launches, err);
    }
    for (int sim = 0; sim < N; ++sim) {
        if (teacher) {
            a.net_value = call.teacher.value + sim; a.net_reward = call.teacher.reward + sim;
            a.net_policy = call.teacher.priors + (size_t)sim * A;
            a.value_stride = N; a.policy_stride = N * A; a.policy_is_prior = 1;
        } else {
            InferCall c{};
            c.n = n; c.g0 = call.g0; c.recurrent = 1; c.action = pool.leaf_action; c.gather_parent = pool.leaf_parent;
            c.pool_hidden = pool.hidden; c.pool_stride = NP + 1; c.out_slot = (K0 > 0 ? K0 : 1) + sim;
            c.value = pool.net_value; c.reward = pool.net_reward; c.policy_logits = pool.net_policy;
            int rc = infer(c);
            if (rc) return rc;
            a.net_value = pool.net_value; a.net_reward = pool.net_reward; a.net_policy = pool.net_policy;
            a.value_stride = 1; a.policy_stride = A; a.policy_is_prior = 0;
        }
        a.sim = sim + 1; a.do_root = 0; a.do_update = 1; a.do_select = (sim + 1 < N); a.do_final = (sim + 1 == N);
        kt_begin(KT_TREE, stream);
        e = launch_tree_step(a, stream);
        kt_end(stream);
        if (e != cudaSuccess) return cuda_fail("tree_step", e);
        *launches += 1;
    }
    return MZ_OK;
}

}  // namespace mz
