// Persistent fused search kernel for fully-connected MuZero networks.
//
// One launch runs the reference's whole MCTS.run (self_play.py:260-361) - root inference,
// root expansion + Dirichlet mixing, N x {select, recurrent inference, support_to_scalar,
// expand, backup} - for every game of the batch.  A group of G lanes owns one game from the
// first to the last simulation: its tree (child slots, hidden states, path) lives in shared
// memory next to the network weights, so the only HBM traffic is the observation in and
// the visit counts / root values out.  The groups of a warp share its collectives (common.cuh,
// LaneGroup), warps never synchronise with each other; the grid is persistent (one wave) and warps stride over the games.
#include "fc_net.cuh"
#include "tree.cuh"
#include "kernels.h"

#include <stdlib.h>
#include <algorithm>
#include <vector>

namespace mz {

struct GameSmem {
    // byte offsets inside one game's region
    int vsum, mval, root_prior, visit, expansion, reward, prior, path, path_reward, hidden, act, bytes;
};

__host__ __device__ inline GameSmem game_smem_layout(int N, int A, int E, int maxw, bool keep_hidden) {
    GameSmem L;
    const int S = (N + 1) * A;
    const int Epad = (E + 3) & ~3;
    int off = 0;
    auto take = [&](int bytes) { int o = off; off = (off + bytes + 15) & ~15; return o; };
    L.vsum = take(S * 8);
    L.mval = take(S * 8);
    L.root_prior = take(A * 8);
    L.visit = take(S * 4);
    L.expansion = take(S * 4);
    L.reward = take(S * 4);
    L.prior = take(S * 4);
    L.path = take((N + 2) * 4);
    L.path_reward = take((N + 2) * 4);
    L.hidden = take((keep_hidden ? (N + 1) * Epad : 0) * 4);
    L.act = take(9 * maxw * 4);        // s0 s1 s2 + three heads x (ping, pong)
    off += 16;          // odd multiple of 16 B between games: spreads games over banks
    L.bytes = off;
    return L;
}

// Phase split (scripts/fc_phase_split.py builds a copy of the library with -DMZ_FC_PHASES): every group times its game's
// root, select, network, expand and backup phases with clock() and adds them, with the levels and selection rounds it
// walked, to device counters that mz_fc_phase_counters reads.  It also stores the %globaltimer at which its game started
// and finished (mz_fc_phase_spans): games that start after others have finished ran in a later pass of the persistent
// loop, and the SM it ran on (%smid; mz_fc_phase_rows reads whole rows).  The library built without the macro is unchanged.
enum { kPhRoot, kPhSelect, kPhNet, kPhExpand, kPhBackup, kPhLevels, kPhRounds, kPhSims, kPhSums,
       kPhStart = kPhSums, kPhEnd, kPhSm, kPhCount };
// The counters are per game and added to in memory as the game goes (fire-and-forget reductions to distinct addresses):
// accumulators held in registers would push the kernel past 128 registers and change its occupancy.  The start and end
// times sit in the same row.
#ifdef MZ_FC_PHASES
constexpr int kPhMaxGames = 1 << 16;
__device__ unsigned long long g_fc_phase[kPhMaxGames][kPhCount];
MZ_DEVINL unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
struct PhaseClock {
    int row = -1;                     // game of this group's lane 0, -1 on the other lanes
    unsigned last = 0;
    MZ_DEVINL void start(int g, bool leader) {
        row = (leader && g < kPhMaxGames) ? g : -1;
        if (row >= 0) atomicExch(&g_fc_phase[row][kPhStart], global_ns());
        last = (unsigned)clock();
    }
    // an exchange, like the counters' reductions, leaves the kernel without spills where a plain store did not
    MZ_DEVINL void finish() {
        if (row < 0) return;
        unsigned sm;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
        atomicExch(&g_fc_phase[row][kPhEnd], global_ns());
        atomicExch(&g_fc_phase[row][kPhSm], (unsigned long long)sm);
    }
    MZ_DEVINL void mark(int p) {
        const unsigned now = (unsigned)clock();
        if (row >= 0) atomicAdd(&g_fc_phase[row][p], (unsigned long long)(now - last));
        last = now;
    }
    MZ_DEVINL void count(int p, int n) { if (row >= 0) atomicAdd(&g_fc_phase[row][p], (unsigned long long)n); }
};
// %globaltimer at which each CTA entered the kernel, before it stages the tables and weights (mz_fc_phase_ctas)
constexpr int kPhMaxCtas = 1 << 14;
__device__ unsigned long long g_fc_cta_entry[kPhMaxCtas];
MZ_DEVINL void phase_cta_entry() { if (threadIdx.x == 0 && blockIdx.x < kPhMaxCtas) g_fc_cta_entry[blockIdx.x] = global_ns(); }
#else
struct PhaseClock {
    MZ_DEVINL void start(int, bool) {}
    MZ_DEVINL void finish() {}
    MZ_DEVINL void mark(int) {}
    MZ_DEVINL void count(int, int) {}
};
MZ_DEVINL void phase_cta_entry() {}
#endif

// ---- the search's two network calls (fc_search_kernel and fc_debug_net_kernel run these)
// A tap sees each intermediate vector of a call while it is still in shared memory - tap(what, v, n), v[0..n) - and may only
// read it: the next write to that scratch follows a group barrier.  The search passes NoTap; mz_debug_fc_net copies them out.
enum { kTapRaw, kTapReward, kTapPolicy, kTapValue };
struct NoTap { MZ_DEVINL void operator()(int, const float*, int) const {} };

// Root: representation (models.py:133-145) of obs into hidden (rescaled, zero padded to a multiple of 4), then prediction
// (models.py:128-131): this lane's policy logit (0 in lanes >= A) and the scalarised value.  s0, s1, s2: scratch of maxw.
// E and S are the kernel's net.E and net.S, read once per launch: re-reading them through `net` here changes the search
// kernel's code (fc_search_kernel's SASS is the same as with these blocks written inline).
template <int G, typename Tap>
MZ_DEVINL void fc_root_inference(const FcNet& net, const float* blob, const float* obs, float* hidden, float* s0, float* s1,
                                 float* s2, int E, int S, int A, float& logit, float& value, Tap&& tap) {
    const int lane = LaneGroup<G>::lane();
    load_vector<G>(obs, s1, net.obs_elems);
    float* raw = mlp_forward<G>(net.rep, blob, s1, s0, s1, s2);
    tap(kTapRaw, raw, E);
    rescale_unit_range<G>(raw, hidden, E);
    float* pol = mlp_forward<G>(net.pol, blob, hidden, s0, s1, s2);
    logit = (lane < A) ? pol[lane] : 0.0f;
    tap(kTapPolicy, pol, A);
    LaneGroup<G>::sync();
    float* val = mlp_forward<G>(net.val, blob, hidden, s0, s1, s2);
    value = support_to_scalar_group<G>(val, S);
    tap(kTapValue, val, 2 * S + 1);
    LaneGroup<G>::sync();
}

// One simulation's recurrent inference (models.py:147-170, 128-131): dynamics of (h, action) into hn (rescaled, zero padded),
// this lane's prior (softmax over the first A lanes), the scalarised value and reward.  SH = FcFixedShape runs the unrolled
// fc_recurrent_fixed; otherwise the descriptors walk, with the three heads side by side (mlp_forward_multi) when they have
// equal depth (fused_heads) and one after the other when not.  hb: the heads' ping-pong vectors, 3 x 2 of maxw.
template <int G, typename SH, typename Tap>
MZ_DEVINL void fc_sim_inference(const FcNet& net, const float* blob, const float* h, int action, float* hn, float* s0, float* s1,
                                float* s2, float* const (&hb)[3][2], bool fused_heads, int E, int S, int A, float& logit,
                                float& prior, float& value, float& reward, Tap&& tap) {
    const int lane = LaneGroup<G>::lane();
    const int F = 2 * S + 1;
    if constexpr (SH::kEnabled) {
        fc_recurrent_fixed<G, SH>(net, blob, h, action, hn, s0, s1, hb[0][0], hb[1][0], hb[2][0], prior, value, reward);
        tap(kTapRaw, s1, E);                            // the logits stay in registers
    } else {
        float* raw = mlp_forward<G>(net.dyn, blob, h, s0, s1, s2, action);
        if (fused_heads) {
            // rescale first, then reward (raw state), policy and value (rescaled state) side by side
            rescale_unit_range<G>(raw, hn, E);
            const MlpDesc* const ds[3] = {&net.rew, &net.pol, &net.val};
            const float* const xs[3] = {raw, hn, hn};
            float* outs[3];
            mlp_forward_multi<G, 3>(ds, blob, xs, hb, outs);
            logit = (lane < A) ? outs[1][lane] : 0.0f;
            support_to_scalar_group2<G>(outs[2], outs[0], S, value, reward);
            tap(kTapRaw, raw, E); tap(kTapReward, outs[0], F); tap(kTapPolicy, outs[1], A); tap(kTapValue, outs[2], F);
            LaneGroup<G>::sync();
        } else {
            // reward head reads the un-normalised next state
            float* rl = mlp_forward<G>(net.rew, blob, raw, s0, s1, nullptr);
            reward = support_to_scalar_group<G>(rl, S);
            tap(kTapRaw, raw, E); tap(kTapReward, rl, F);
            LaneGroup<G>::sync();
            rescale_unit_range<G>(raw, hn, E);
            float* pol = mlp_forward<G>(net.pol, blob, hn, s0, s1, s2);
            logit = (lane < A) ? pol[lane] : 0.0f;
            tap(kTapPolicy, pol, A);
            LaneGroup<G>::sync();
            float* vl = mlp_forward<G>(net.val, blob, hn, s0, s1, s2);
            value = support_to_scalar_group<G>(vl, S);
            tap(kTapValue, vl, F);
            LaneGroup<G>::sync();
        }
        prior = group_softmax_masked<G>(logit, lane < A);
    }
}

// global -> shared copies that do not pass through registers (cp.async, sm_80+); cp_async_wait_all waits for the thread's own
MZ_DEVINL void cp_async8(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
MZ_DEVINL void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
MZ_DEVINL void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <typename SH>
constexpr int fixed_actions() {
    if constexpr (SH::kEnabled) return SH::A;
    else return 0;
}

// SH: FcFixedShape<E, H, S, A> runs the per-simulation network call through the fully unrolled fixed-shape code
// (fc_net.cuh::fc_recurrent_fixed, bit-identical to the generic descriptors walk), FcGenericShape through the latter.
// The fixed shape also fixes the tree's action count; kP is the number of players when fixed at compile time (0 = a.P).
template <int G, bool kTeacher, typename SH, int kP>
__global__ void __launch_bounds__(kFcMaxThreads, 2) fc_search_kernel(const __grid_constant__ FcSearchArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    constexpr int kA = fixed_actions<SH>();
    const int N = a.N, A = kA ? kA : a.A;
    // ---- CTA-shared: tables + weights
    double* s_pbc = reinterpret_cast<double*>(smem);
    double* s_sqrt = s_pbc + (N + 2);
    float* s_blob = reinterpret_cast<float*>(s_sqrt + (N + 2));
    phase_cta_entry();
    // Asynchronous copies (LDGSTS): every thread's share of the tables and the blob is in flight at once, so a CTA waits
    // one global-memory latency (cold: the L2 holds nothing of this launch yet) instead of one per strided iteration.
    // The blob is padded to a multiple of 4 floats in global memory (abi.cu) and starts 16-byte aligned in both spaces;
    // the prefetch brings the first game's observation row in meanwhile.
    if (!kTeacher && (threadIdx.x & (G - 1)) == 0) {
        const int g = min((int)blockIdx.x * (int)(blockDim.x / G) + (int)threadIdx.x / G, a.n_games - 1);
        asm volatile("prefetch.global.L1 [%0];" ::"l"(a.obs + (size_t)g * a.net.obs_elems));
    }
    for (int i = threadIdx.x; i < N + 2; i += blockDim.x) { cp_async8(s_pbc + i, a.pbc + i); cp_async8(s_sqrt + i, a.sqrtn + i); }
    if (!kTeacher)
        for (int i = threadIdx.x; i < (a.net.blob_floats + 3) >> 2; i += blockDim.x) cp_async16(s_blob + 4 * i, a.blob + 4 * i);
    cp_async_wait_all();
    __syncthreads();

    const int shared_bytes = ((2 * (N + 2) * 8 + (kTeacher ? 0 : a.net.blob_floats) * 4) + 15) & ~15;
    const GameSmem L = game_smem_layout(N, A, a.net.E, a.net.maxw, !kTeacher);
    const int groups_per_cta = blockDim.x / G;
    const int gi = threadIdx.x / G;
    const int lane = LaneGroup<G>::lane();
    unsigned char* mine = smem + shared_bytes + (size_t)gi * L.bytes;

    TreeConst c;
    c.A = A; c.N = N; c.P = a.P; c.discount = a.discount; c.noise_frac = a.noise_frac; c.noise_alpha = a.noise_alpha; c.seed = a.seed;
    c.pbc = s_pbc; c.sqrtn = s_sqrt; c.ucb = a.ucb;

    GameTree t;
    t.vsum = reinterpret_cast<double*>(mine + L.vsum);
    t.mval = reinterpret_cast<double*>(mine + L.mval);
    t.root_prior = reinterpret_cast<double*>(mine + L.root_prior);
    t.visit = reinterpret_cast<int*>(mine + L.visit);
    t.expansion = reinterpret_cast<int*>(mine + L.expansion);
    t.reward = reinterpret_cast<float*>(mine + L.reward);
    t.prior = reinterpret_cast<float*>(mine + L.prior);
    t.path = reinterpret_cast<int*>(mine + L.path);
    t.path_reward = reinterpret_cast<float*>(mine + L.path_reward);
    float* s_hidden = reinterpret_cast<float*>(mine + L.hidden);
    float* s_act = reinterpret_cast<float*>(mine + L.act);
    const int E = a.net.E, S = a.net.S, maxw = a.net.maxw;
    const int Epad = (E + 3) & ~3;
    float* s0 = s_act;
    float* s1 = s_act + maxw;
    float* s2 = s_act + 2 * maxw;
    float* const hb[3][2] = {{s_act + 3 * maxw, s_act + 4 * maxw}, {s_act + 5 * maxw, s_act + 6 * maxw},
                             {s_act + 7 * maxw, s_act + 8 * maxw}};
    const bool fused_heads = (a.net.rew.n == a.net.pol.n) && (a.net.pol.n == a.net.val.n);
    // multi-level selection: A fixed at compile time for the fixed network shapes
    constexpr int kMaxD = select_levels_for(kA ? kA : 2, G);
    const SelectLanes sl = select_lanes<G, kA>(A, min(a.select_levels, kMaxD));
    PhaseClock ph;

    // The warp's groups run their games side by side (see LaneGroup): the loop goes on while the warp's first group has a
    // game, and a group past the last game searches that one again (it belongs to this warp) and stores nothing.
    const int warp_first = (int)blockIdx.x * groups_per_cta + (int)(threadIdx.x & ~31u) / G;
    for (int g0 = warp_first; g0 < a.n_games; g0 += gridDim.x * groups_per_cta) {
        const int g_own = g0 + gi - (int)(threadIdx.x & ~31u) / G;
        const bool own = g_own < a.n_games;
        const int g = own ? g_own : a.n_games - 1;
        ph.start(g, lane == 0 && own);
        const int64_t game_id = a.game_id ? a.game_id[g] : (int64_t)g;
        const int move = a.move_index ? a.move_index[g] : 0;
        const int to_play0 = a.to_play ? a.to_play[g] : 0;
        const int first_index = a.first_index ? a.first_index[g] : -1;
        unsigned legal = 0;
        for (int k = 0; k < A; ++k) legal |= (a.legal_mask == nullptr || a.legal_mask[(size_t)g * A + k]) ? (1u << k) : 0u;
        t.legal = legal;
        (void)to_play0;

        // ------------------------------------------------------------------ root
        float root_value, root_reward, logit = 0.0f;
        if (kTeacher) {
            root_value = a.teacher.root_value[g];
            root_reward = a.teacher.root_reward[g];
        } else {
            fc_root_inference<G>(a.net, s_blob, a.obs + (size_t)g * a.net.obs_elems, s_hidden, s0, s1, s2, E, S, A, logit, root_value,
                                 NoTap{});
            root_reward = inverse_value_transform(0.0f);     // log(one-hot centre), models.py:176-183
        }
        float prior;
        if (kTeacher) prior = (lane < A) ? a.teacher.root_priors[(size_t)g * A + lane] : 0.0f;
        else prior = group_softmax_masked<G>(logit, lane < A && ((legal >> lane) & 1u));
        if (a.trace.root_priors_raw && lane < A && own) a.trace.root_priors_raw[(size_t)g * A + lane] = ((legal >> lane) & 1u) ? prior : 0.0f;
        if (a.trace.root_reward && lane == 0 && own) a.trace.root_reward[g] = root_reward;
        tree_init_root<G, kA>(c, t, prior, root_reward,
                              (a.add_noise && a.noise) ? a.noise + (size_t)g * A : nullptr, a.add_noise && !a.noise,
                              game_id, move, (a.trace.noise && own) ? a.trace.noise + (size_t)g * A : nullptr);
        ph.mark(kPhRoot);

        // ------------------------------------------------------------------ simulations
        int max_depth = 0;
        // every path through a simulation ends converged (the backup's REDUX waits for the warp), so with the loop entered
        // converged ptxas proves each of its collectives and emits no divergence test (LaneGroup::converge)
        LaneGroup<G>::converge();
        for (int sim = 0; sim < N; ++sim) {
            int rounds;
            const Leaf leaf = tree_select_lookahead<G, kMaxD, kA>(c, t, sl, sim, game_id, move, first_index, rounds);
            ph.mark(kPhSelect);
            ph.count(kPhLevels, leaf.depth);
            ph.count(kPhRounds, rounds);
            float value, reward;
            if (kTeacher) {
                value = a.teacher.value[(size_t)g * N + sim];
                reward = a.teacher.reward[(size_t)g * N + sim];
                prior = (lane < A) ? a.teacher.priors[((size_t)g * N + sim) * A + lane] : 0.0f;
            } else {
                fc_sim_inference<G, SH>(a.net, s_blob, s_hidden + (size_t)leaf.parent_exp * Epad, leaf.action,
                                        s_hidden + (size_t)t.n_expanded * Epad, s0, s1, s2, hb, fused_heads, E, S, A, logit, prior, value, reward,
                                        NoTap{});
            }
            ph.mark(kPhNet);
            if (a.trace.depth && own) {
                const size_t ti = (size_t)g * N + sim;
                if (lane == 0) { a.trace.depth[ti] = leaf.depth; a.trace.value[ti] = value; a.trace.reward[ti] = reward; }
                if (lane < A) a.trace.priors[ti * A + lane] = prior;
                for (int j = lane; j < leaf.depth && j < a.trace.max_depth; j += G)
                    a.trace.actions[ti * a.trace.max_depth + j] = (uint8_t)(t.path[j + 1] % A);
            }
            tree_expand<G, kA>(c, t, leaf, reward, prior);
            ph.mark(kPhExpand);
            tree_backup<G, kP, true>(c, t, leaf, value);
            ph.mark(kPhBackup);
            max_depth = max(max_depth, leaf.depth);
        }
        ph.count(kPhSims, N);

        // ------------------------------------------------------------------ results
        if (lane < A && own) {
            const bool ok = (legal >> lane) & 1u;
            if (a.visit_counts) a.visit_counts[(size_t)g * A + lane] = ok ? t.visit[lane] : 0;
            if (a.root_priors) a.root_priors[(size_t)g * A + lane] = t.root_prior[lane];
        }
        if (lane == 0 && own) {
            if (a.root_value) a.root_value[g] = (t.root_visit == 0) ? 0.0 : __ddiv_rn(t.root_vsum, (double)t.root_visit);
            if (a.root_predicted_value) a.root_predicted_value[g] = root_value;
            if (a.max_tree_depth) a.max_tree_depth[g] = max_depth;
            if (a.tie_count) a.tie_count[g] = t.ties;
            if (a.value_range) { a.value_range[2 * g] = t.lo; a.value_range[2 * g + 1] = t.hi; }
        }
        if (a.pool.visit && own) {      // MZ_FLAG_KEEP_TREE: spill the shared-memory tree to the HBM node pool
            const int slots = (N + 1) * A;
            const size_t pb = (size_t)g * slots;
            for (int s = lane; s < t.n_expanded * A; s += G) {
                a.pool.visit[pb + s] = t.visit[s];
                a.pool.vsum[pb + s] = t.vsum[s];
                a.pool.reward[pb + s] = t.reward[s];
                a.pool.prior[pb + s] = t.prior[s];
                a.pool.expansion[pb + s] = t.expansion[s];
            }
            if (lane < A) a.pool.root_prior[(size_t)g * A + lane] = t.root_prior[lane];
            if (!kTeacher && a.pool.hidden)
                for (int i = lane; i < t.n_expanded * E; i += G)
                    a.pool.hidden[(size_t)g * (N + 1) * E + i] = s_hidden[(i / E) * Epad + (i % E)];
            if (lane == 0) {
                a.pool.root_visit[g] = t.root_visit;
                a.pool.root_vsum[g] = t.root_vsum;
                a.pool.n_expanded[g] = t.n_expanded;
            }
        }
        ph.finish();
        LaneGroup<G>::sync();
    }
}

// ------------------------------------------------------------------------------------------
// host launcher
// ------------------------------------------------------------------------------------------
// Shared memory of a CTA of `groups` games: the UCB tables and (student kernels) the weight blob, then one region per game.
static size_t fc_cta_smem(int N, int A, int E, int maxw, int blob_floats, bool teacher, int groups) {
    const GameSmem L = game_smem_layout(N, A, E, maxw, !teacher);
    const size_t shared_bytes = ((2 * (size_t)(N + 2) * 8 + (teacher ? 0 : (size_t)blob_floats) * 4) + 15) & ~(size_t)15;
    return shared_bytes + (size_t)groups * L.bytes;
}

// The kernel is latency-bound: a game's chain of dependent simulations barely lengthens with the number of games that
// share its SM, so the launch lasts about one chain per pass and the plan minimises passes.  Resident CTAs per SM follow
// the occupancy rules of sm_90: shared memory in 128-byte units plus the per-CTA reserve, registers in 256-register
// units per warp out of 64K, at most 2048 threads and 32 CTAs.
bool fc_search_plan(int N, int A, int E, int maxw, int blob_floats, int G, bool teacher, int n_games, int sm_count,
                    size_t smem_per_sm, size_t smem_reserve, size_t smem_cap, int regs, int threads, FcPlan* plan) {
    if (n_games < 1 || sm_count < 1 || G < 1 || regs < 1 || N < 0 || A < 1 || E < 1 || maxw < 1 || blob_floats < 0) return false;
    bool found = false;
    const std::vector<int> sizes = threads != 0 ? std::vector<int>{threads} : std::vector<int>{64, 128, 256};
    for (int t : sizes) {
        if (t % 32 != 0 || t < G || t > kFcMaxThreads) continue;
        const int groups = t / G;
        const size_t smem = fc_cta_smem(N, A, E, maxw, blob_floats, teacher, groups);
        const int by_smem = smem > smem_cap ? 0 : (int)(smem_per_sm / ((smem + smem_reserve + 127) & ~(size_t)127));
        const int by_regs = (65536 / (((regs * 32) + 255) & ~255)) / (t / 32);
        const int per_sm = std::min(std::min(by_smem, by_regs), std::min(2048 / t, 32));
        if (per_sm >= 1) {
            const int slots = per_sm * groups * sm_count;
            const int passes = (n_games + slots - 1) / slots;
            if (!found || passes < plan->passes) {
                *plan = FcPlan{t, groups, per_sm, slots, passes, smem};
                found = true;
            }
        }
    }
    return found;
}

template <int G, bool T, typename SH, int kP>
static cudaError_t launch_kernel(const FcSearchArgs& a, const FcLaunchInfo& l, cudaStream_t stream) {
    fc_search_kernel<G, T, SH, kP><<<l.grid, l.block, l.smem, stream>>>(a);
    return cudaGetLastError();
}

// Picks the launch of instantiation <G, T, SH, kP> for a.n_games games into *p: selection levels, plan and grid.
template <int G, bool T, typename SH, int kP = 0>
static cudaError_t prepare_one(const FcSearchArgs& a, bool one_level, int sm_count, FcLaunchState* st, FcPrepared* p) {
    p->select_levels = one_level ? 1 : select_levels_for(a.A, G);
    auto kern = fc_search_kernel<G, T, SH, kP>;
    const void* fn = reinterpret_cast<const void*>(kern);
    int regs = 0;
    for (const auto& k : st->kernels) if (k.fn == fn) regs = k.regs;
    if (regs == 0) {
        // the driver's default carveout may leave less shared memory per SM than the plan counts on
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)st->smem_cap);
        if (err == cudaSuccess) err = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncAttributes fa{};
        if (err == cudaSuccess) err = cudaFuncGetAttributes(&fa, kern);
        if (err != cudaSuccess) return err;
        regs = fa.numRegs;
        st->kernels.push_back({fn, regs});
    }
    FcPlan plan;
    if (!fc_search_plan(a.N, a.A, a.net.E, a.net.maxw, a.net.blob_floats, G, T, a.n_games, sm_count, st->smem_per_sm,
                        st->smem_reserve, st->smem_cap, regs, a.threads, &plan))
        return cudaErrorInvalidConfiguration;
    int per_sm = -1;
    for (const auto& s : st->shapes) if (s.fn == fn && s.threads == plan.threads && s.smem == plan.smem) per_sm = s.ctas_per_sm;
    if (per_sm < 0) {
        cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, plan.threads, plan.smem);
        if (err != cudaSuccess) return err;
        st->shapes.push_back({fn, plan.threads, plan.smem, per_sm});
    }
    per_sm = std::min(per_sm, plan.ctas_per_sm);      // the device's word when it disagrees with the plan
    if (per_sm < 1) return cudaErrorInvalidConfiguration;
    const int want = (a.n_games + plan.groups - 1) / plan.groups;
    const int grid = std::min(want, per_sm * sm_count);
    p->launch = launch_kernel<G, T, SH, kP>;
    p->fixed_shape = SH::kEnabled;
    p->info = FcLaunchInfo{grid, plan.threads, per_sm, G, plan.smem};
    return cudaSuccess;
}

// shapes with a fully unrolled network path: games/cartpole.py (encoding 8, hidden 16, support 10, 2 actions)
using CartPoleShape = FcFixedShape<8, 16, 10, 2>;

// Does the search run the unrolled network of CartPoleShape at this lane-group width?
static bool fc_uses_fixed(const FcNet& net, int G) { return (G == 16 || G == 32) && fc_matches_fixed<CartPoleShape>(net); }

static cudaError_t prepare_fc_search(const FcSearchArgs& a, int group, bool teacher, bool generic, bool one_level,
                                     int sm_count, FcLaunchState* st, FcPrepared* p) {
    if (!teacher && !generic && fc_uses_fixed(a.net, group)) {
        // (a single player: the backup's value recurrence and its signs simplify)
        if (group == 16 && a.P == 1) return prepare_one<16, false, CartPoleShape, 1>(a, one_level, sm_count, st, p);
        if (group == 16) return prepare_one<16, false, CartPoleShape>(a, one_level, sm_count, st, p);
        if (group == 32 && a.P == 1) return prepare_one<32, false, CartPoleShape, 1>(a, one_level, sm_count, st, p);
        if (group == 32) return prepare_one<32, false, CartPoleShape>(a, one_level, sm_count, st, p);
    }
#define MZ_CASE(GG)                                                                                     \
    case GG:                                                                                            \
        return teacher ? prepare_one<GG, true, FcGenericShape>(a, one_level, sm_count, st, p)           \
                       : prepare_one<GG, false, FcGenericShape>(a, one_level, sm_count, st, p);
    switch (group) {
        MZ_CASE(4)
        MZ_CASE(8)
        MZ_CASE(16)
        MZ_CASE(32)
    }
#undef MZ_CASE
    return cudaErrorInvalidValue;
}

cudaError_t launch_fc_search(const FcSearchArgs& a_in, int group, bool teacher, int sm_count, FcLaunchState* st,
                             cudaStream_t stream) {
    // A/B switches, read per launch so that a caller may flip them between searches of one handle:
    // MZ_FC_GENERIC=1 always walks the layer descriptors, MZ_FC_SELECT_LEVELS=1 resolves one tree level per round
    const char* generic = getenv("MZ_FC_GENERIC");
    const char* levels = getenv("MZ_FC_SELECT_LEVELS");
    FcPreparedKey key{a_in.n_games, group, a_in.threads, teacher, generic && generic[0] == '1',
                      levels && levels[0] == '1' && levels[1] == 0};
    FcPrepared& p = st->prepared;
    if (!p.valid || !(p.key == key)) {
        p.valid = false;
        const cudaError_t err = prepare_fc_search(a_in, group, teacher, key.generic, key.one_level, sm_count, st, &p);
        if (err != cudaSuccess) return err;
        p.key = key;
        p.valid = true;
    }
    FcSearchArgs a = a_in;
    a.select_levels = p.select_levels;
    const cudaError_t err = p.launch(a, p.info, stream);
    if (err == cudaSuccess) {
        st->launched = true;
        st->last = p.info;
    }
    return err;
}

// ------------------------------------------------------------------------------------------
// mz_debug_fc_net: the network calls of the search and of fc_inference_kernel on their own
// ------------------------------------------------------------------------------------------
// Copies each tapped vector of the group's sample to global memory (the rows of samples past the last one stay untouched).
struct CopyTap {
    const FcDebugArgs* a;
    int g, lane, step;
    bool own;
    MZ_DEVINL void operator()(int what, const float* v, int n) const {
        float* dst = what == kTapRaw ? a->raw : what == kTapReward ? a->reward_logits : what == kTapPolicy ? a->policy_logits : a->value_logits;
        if (!dst || !own) return;
        for (int i = lane; i < n; i += step) dst[(size_t)g * n + i] = v[i];
    }
};

// The search's root evaluation or one simulation's network call for each of a.n samples, with the shared-memory layout of
// fc_search_kernel (the blob, then per game the region of game_smem_layout, here for a one-simulation tree), every game's
// region overwritten with NaN bytes before the first layer.  One warp per CTA; the groups stride over the samples as in the
// search.  force_split walks the descriptors with the heads one after the other even for the fixed shape or heads of equal
// depth (the network never does).
template <int G, typename SH>
__global__ void __launch_bounds__(32) fc_debug_net_kernel(const __grid_constant__ FcDebugArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    float* s_blob = reinterpret_cast<float*>(smem);
    for (int i = threadIdx.x; i < a.net.blob_floats; i += blockDim.x) s_blob[i] = a.blob[i];
    __syncthreads();
    const int E = a.net.E, A = a.net.A, maxw = a.net.maxw, Epad = (E + 3) & ~3;
    const GameSmem L = game_smem_layout(1, A, E, maxw, true);
    const int groups_per_cta = blockDim.x / G;
    const int gi = threadIdx.x / G;
    const int lane = LaneGroup<G>::lane();
    unsigned char* mine = smem + ((a.net.blob_floats * 4 + 15) & ~15) + (size_t)gi * L.bytes;
    float* s_hidden = reinterpret_cast<float*>(mine + L.hidden);
    float* s_act = reinterpret_cast<float*>(mine + L.act);
    float* s0 = s_act;
    float* s1 = s_act + maxw;
    float* s2 = s_act + 2 * maxw;
    float* const hb[3][2] = {{s_act + 3 * maxw, s_act + 4 * maxw}, {s_act + 5 * maxw, s_act + 6 * maxw},
                             {s_act + 7 * maxw, s_act + 8 * maxw}};
    const bool fused_heads = (a.net.rew.n == a.net.pol.n) && (a.net.pol.n == a.net.val.n) && !a.force_split;
    const int warp_first = (int)blockIdx.x * groups_per_cta + (int)(threadIdx.x & ~31u) / G;
    for (int g0 = warp_first; g0 < a.n; g0 += gridDim.x * groups_per_cta) {
        const int g_own = g0 + gi - (int)(threadIdx.x & ~31u) / G;
        const bool own = g_own < a.n;
        const int g = own ? g_own : a.n - 1;
        for (int i = lane; i < L.bytes / 4; i += G) reinterpret_cast<unsigned*>(mine)[i] = 0xFFFFFFFFu;
        LaneGroup<G>::sync();
        const CopyTap tap{&a, g, lane, G, own};
        float logit = 0.0f, prior, value, reward = 0.0f;
        float* hn = s_hidden;
        if (a.route == MZ_FC_SEARCH_ROOT) {
            fc_root_inference<G>(a.net, s_blob, a.in + (size_t)g * a.net.obs_elems, s_hidden, s0, s1, s2, E, a.net.S, A, logit, value,
                                 tap);
            prior = group_softmax_masked<G>(logit, lane < A);
        } else {
            load_vector<G>(a.in + (size_t)g * E, s_hidden, E);
            hn = s_hidden + Epad;
            fc_sim_inference<G, SH>(a.net, s_blob, s_hidden, a.action[g], hn, s0, s1, s2, hb, fused_heads, E, a.net.S, A, logit, prior, value,
                                    reward, tap);
        }
        if (own) {
            if (a.hidden) for (int i = lane; i < E; i += G) a.hidden[(size_t)g * E + i] = hn[i];
            if (a.prior && lane < A) a.prior[(size_t)g * A + lane] = prior;
            if (lane == 0) {
                if (a.value) a.value[g] = value;
                if (a.reward && a.route == MZ_FC_SEARCH_SIM) a.reward[g] = reward;
            }
        }
        LaneGroup<G>::sync();
    }
}

bool fc_debug_plan(const FcNet& net, int G, int route, bool force_split, int n, int sm_count, size_t smem_cap, int64_t* plan,
                   std::string* err) {
    if (G != 4 && G != 8 && G != 16 && G != 32) { *err = "the lane group must be 4, 8, 16 or 32"; return false; }
    if (n < 1 || sm_count < 1) { *err = "bad batch or SM count"; return false; }
    if (route == MZ_FC_INFER_INITIAL || route == MZ_FC_INFER_RECURRENT || route == MZ_FC_INFER_POOL) {
        FcInferPlan p;
        if (!fc_infer_plan(net.blob_floats, net.maxw, G, n, sm_count, smem_cap, &p)) {
            *err = "fc_inference_kernel needs " + std::to_string(fc_infer_smem(net.blob_floats, net.maxw, 32 / G)) +
                   " bytes of shared memory for one warp, the device allows " + std::to_string(smem_cap);
            return false;
        }
        const int64_t out[5] = {MZ_FC_PATH_INFER, G, p.threads, p.grid, (int64_t)p.smem};
        for (int i = 0; i < 5; ++i) plan[i] = out[i];
        return true;
    }
    if (route != MZ_FC_SEARCH_ROOT && route != MZ_FC_SEARCH_SIM) { *err = "unknown route"; return false; }
    if (net.A > G) { *err = "the search needs one lane per action (action_space <= lane group)"; return false; }
    const bool fixed = fc_uses_fixed(net, G) && !force_split;
    const bool fused = net.rew.n == net.pol.n && net.pol.n == net.val.n && !force_split;
    const GameSmem L = game_smem_layout(1, net.A, net.E, net.maxw, true);
    const size_t smem = (size_t)((net.blob_floats * 4 + 15) & ~15) + (size_t)(32 / G) * L.bytes;
    if (smem > smem_cap) {
        *err = "the search's network call needs " + std::to_string(smem) + " bytes of shared memory, the device allows " +
               std::to_string(smem_cap);
        return false;
    }
    const int groups = 32 / G;
    const int grid = std::min((n + groups - 1) / groups, 8 * sm_count);
    const int64_t out[5] = {fixed ? MZ_FC_PATH_FIXED : fused ? MZ_FC_PATH_FUSED : MZ_FC_PATH_SPLIT, G, 32, grid, (int64_t)smem};
    for (int i = 0; i < 5; ++i) plan[i] = out[i];
    return true;
}

template <int G, typename SH>
static cudaError_t launch_debug(const FcDebugArgs& a, int grid, size_t smem, cudaStream_t stream) {
    auto kern = fc_debug_net_kernel<G, SH>;
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
    kern<<<grid, 32, smem, stream>>>(a);
    return cudaGetLastError();
}

// the search routes of mz_debug_fc_net (plan from fc_debug_plan)
cudaError_t launch_fc_debug_net(const FcDebugArgs& a, int G, const int64_t* plan, cudaStream_t stream) {
    const int grid = (int)plan[3];
    const size_t smem = (size_t)plan[4];
    if (plan[0] == MZ_FC_PATH_FIXED) {
        if (G == 16) return launch_debug<16, CartPoleShape>(a, grid, smem, stream);
        if (G == 32) return launch_debug<32, CartPoleShape>(a, grid, smem, stream);
        return cudaErrorInvalidValue;
    }
    switch (G) {
        case 4: return launch_debug<4, FcGenericShape>(a, grid, smem, stream);
        case 8: return launch_debug<8, FcGenericShape>(a, grid, smem, stream);
        case 16: return launch_debug<16, FcGenericShape>(a, grid, smem, stream);
        case 32: return launch_debug<32, FcGenericShape>(a, grid, smem, stream);
    }
    return cudaErrorInvalidValue;
}

#ifdef MZ_FC_PHASES
// counters of the phase-split build: out[kPhCount] = root, select, network, expand, backup cycles, levels, rounds,
// simulations, each summed over games; reset != 0 zeroes them afterwards
extern "C" int mz_fc_phase_counters(unsigned long long* out, int reset) {
    cudaError_t e = cudaDeviceSynchronize();
    void* dev = nullptr;
    if (e == cudaSuccess) e = cudaGetSymbolAddress(&dev, g_fc_phase);
    if (e == cudaSuccess && out) {
        std::vector<unsigned long long> rows((size_t)kPhMaxGames * kPhCount);
        e = cudaMemcpy(rows.data(), dev, rows.size() * 8, cudaMemcpyDeviceToHost);
        for (int p = 0; p < kPhSums; ++p) out[p] = 0;
        for (size_t i = 0; i < rows.size(); ++i) if (i % kPhCount < kPhSums) out[i % kPhCount] += rows[i];
    }
    if (e == cudaSuccess && reset) e = cudaMemset(dev, 0, sizeof(g_fc_phase));
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return e == cudaSuccess ? 0 : (int)e;
}

// out[2 * g], out[2 * g + 1] = %globaltimer (ns) at which game g < n of the last launch started and finished (read them
// before mz_fc_phase_counters resets the rows)
extern "C" int mz_fc_phase_spans(unsigned long long* out, int n) {
    if (!out || n < 0 || n > kPhMaxGames) return (int)cudaErrorInvalidValue;
    std::vector<unsigned long long> rows((size_t)n * kPhCount);
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(rows.data(), g_fc_phase, rows.size() * 8);
    for (int g = 0; e == cudaSuccess && g < n; ++g) {
        out[2 * g] = rows[(size_t)g * kPhCount + kPhStart];
        out[2 * g + 1] = rows[(size_t)g * kPhCount + kPhEnd];
    }
    return e == cudaSuccess ? 0 : (int)e;
}

// out[g * cols + c] = column c of game g's row (cycles and counts of kPhRoot..kPhSims, then start ns, end ns, SM), games
// g < n; cols must be the row width (kPhCount)
extern "C" int mz_fc_phase_rows(unsigned long long* out, int n, int cols) {
    if (!out || n < 0 || n > kPhMaxGames || cols != kPhCount) return (int)cudaErrorInvalidValue;
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out, g_fc_phase, (size_t)n * kPhCount * 8);
    return e == cudaSuccess ? 0 : (int)e;
}

// out[b] = %globaltimer (ns) at which CTA b < n of the last launch entered the kernel
extern "C" int mz_fc_phase_ctas(unsigned long long* out, int n) {
    if (!out || n < 0 || n > kPhMaxCtas) return (int)cudaErrorInvalidValue;
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out, g_fc_cta_entry, (size_t)n * 8);
    return e == cudaSuccess ? 0 : (int)e;
}
#endif

}  // namespace mz
