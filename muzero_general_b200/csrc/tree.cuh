// Tree arithmetic of one game, executed by a group of G lanes.
//
// Restates, for the device, the reference's per-simulation tree work:
//   select_child / ucb_score   self_play.py:363-404
//   Node.expand                self_play.py:451-465
//   add_exploration_noise      self_play.py:467-476
//   backpropagate              self_play.py:406-430
//   MinMaxStats                self_play.py:553-570
// All statistics are IEEE fp64 evaluated in the reference's operation order with explicit
// round-to-nearest intrinsics (never contracted into FMAs), so that visit counts, paths and
// root values are bit-identical to the Python implementation when the network outputs are
// the same (teacher / student forcing, tests/test_tree_parity_gpu.py).
//
// Storage (same layout in shared memory for the fused FC kernel and in the HBM node pool):
// expansion e (0 = root, e = i+1 for simulation i) owns the child slots [e*A, e*A+A);
// child k of a non-root expansion is action k; root children are indexed by action id and
// masked by the legal bitmask.  Per slot: visit i32, value_sum f64, reward f32, prior f32,
// expansion id i32 (-1 = leaf).  Root priors after noise are kept in fp64 separately
// (they are not fp32-representable, self_play.py:476).
#pragma once
#include "common.cuh"

namespace mz {

struct TreeConst {
    int A;                 // |action_space|
    int N;                 // num_simulations
    int P;                 // number of players (1 or 2)
    double discount;
    double noise_frac;     // root_exploration_fraction
    double noise_alpha;    // root_dirichlet_alpha (device-generated noise only)
    uint64_t seed;
    const double* pbc;     // [N+2]  log((n+base+1)/base)+init
    const double* sqrtn;   // [N+2]  sqrt(n)
    const double* ucb;     // [(N+2)^2] pbc[n_p] * (sqrtn[n_p] / (n_c + 1)) precomputed by the host, or nullptr
};

// Pointers to ONE game's tree (shared or global memory).
struct GameTree {
    int* visit;            // [(N+1)*A]
    double* vsum;          // [(N+1)*A]
    double* mval;          // [(N+1)*A] reward + discount * (+/-)(value_sum / visits), refreshed by every backup (see tree_backup)
    float* reward;         // [(N+1)*A]
    float* prior;          // [(N+1)*A]
    int* expansion;        // [(N+1)*A]
    double* root_prior;    // [A]
    int* path;             // [N+2] slots of the current simulation, path[0] = -1 (root)
    float* path_reward;    // [N+2] reward of every node on that path (the leaf's entry is filled at expansion)
    // scalars of the game
    int root_visit;
    double root_vsum;
    float root_reward;
    double lo, hi;         // MinMaxStats
    unsigned legal;        // bitmask of legal root actions
    int n_expanded;        // expansions so far (>= 1 after the root expansion)
    int ties;              // exact ties after the first simulation
    bool own = true;       // false: the group has no game and replays a warp neighbour's without storing (see LaneGroup)
};

struct Leaf {
    int depth;             // number of select_child calls
    int parent_exp;        // expansion id of the leaf's parent (its hidden state feeds dynamics)
    int action;            // action leading to the leaf
    int slot;              // child slot of the leaf
};

MZ_DEVINL double value_range_normalize(double v, double lo, double hi) {
    // MinMaxStats.normalize, self_play.py:566-570
    if (hi > lo) {
        // the node that set the lower bound has v == lo: a zero numerator would send the division down its out-of-line
        // slow path (and the whole warp with it); 0 / (hi - lo) is +0, so divide a harmless 1.0 and select
        const double d = __dsub_rn(v, lo);
        const double q = __ddiv_rn(d == 0.0 ? 1.0 : d, __dsub_rn(hi, lo));
        return d == 0.0 ? 0.0 : q;
    }
    return v;
}

// RN(s / n) for an integer 1 <= n < 2^31 from y = RN(1 / n): q0 = RN(s*y), r = s - q0*n, q = RN(q0 + r*y).
// Exact - the same bits as __ddiv_rn(s, n) - whenever s / n is a normal number:
//   * |s*y - s/n| <= 2^-53 |s/n|, so q0 is within 1.5 ulp of s/n.  s and q0*n are multiples of ulp(q0) (s ~ n*q0 has
//     the larger exponent) and |s - q0*n| <= 1.5 n ulp(q0) < 2^53 ulp(q0): the fma's remainder r is exact.
//   * then q0 + r*y = s/n + (1 - n*y)(q0 - s/n), and |1 - n*y| <= 2^-53, so the fma rounds s/n + eta with
//     |eta| <= 3 * 2^-53 ulp(s/n) (a factor 2 covers q0 on the other side of a power of two).
//   * that rounds like s/n unless s/n lies within |eta| of a midpoint m of two doubles.  s and n*m are multiples of
//     ulp(s/n)/2, so a non-zero |s/n - m| = |s - n*m| / n is at least ulp(s/n) / (2n), far above |eta|; and s/n = m
//     would need s = n*m, where m has 54 significant bits and odd n' times it (n = 2^j n') at least as many: no double.
// In the subnormal range exact midpoints exist (9 * 2^-1074 / 6) and this rounding can miss the even neighbour; there,
// and for zero (-0 / n must stay -0), infinite or NaN numerators, the IEEE division runs instead.
MZ_DEVINL double div_by_count(double s, int n, double y) {
    if (!(fabs(s) >= 0x1p-990 && fabs(s) < INFINITY)) return __ddiv_rn(s, (double)n);     // (s / n > 2^-1021 below)
    const double q0 = __dmul_rn(s, y);
    const double r = __fma_rn(-q0, (double)n, s);
    return __fma_rn(r, y, q0);
}

// n-th (0-based) set bit of m
MZ_DEVINL int nth_set_bit(unsigned m, int n) { return (int)__fns(m, 0, n + 1); }

// ------------------------------------------------------------------------------------------
// Root: fp32 softmax over the legal logits, optional Dirichlet mixing.  (self_play.py:460-476)
// `logit` is this lane's policy logit (lane k <-> action k); returns this lane's fp32 prior.
// ------------------------------------------------------------------------------------------
template <int G>
MZ_DEVINL float group_softmax_masked(float logit, bool valid) {
    const float m = group_max_f32<G>(valid ? logit : -INFINITY);
    const float e = valid ? expf(logit - m) : 0.0f;
    const float s = group_sum_f32<G>(e);
    return div_pos_or_zero(e, s);          // masked lanes (e = 0) must not drag the warp through the division slow path
}

// kA: |A| when fixed at compile time (0 = c.A), as in tree_select_lookahead and tree_expand
template <int G, int kA = 0>
MZ_DEVINL void tree_init_root(const TreeConst& c, GameTree& t, float prior_f32, float root_reward,
                              const double* noise /* [A] by action or nullptr */, bool generate_noise = false,
                              int64_t game_id = 0, int move = 0, double* noise_out = nullptr) {
    const int A = kA ? kA : c.A;
    const int k = LaneGroup<G>::lane();
    const bool legal = (k < A) && ((t.legal >> k) & 1u);
    double nz = 0.0;
    bool have_noise = false;
    if (noise != nullptr) {
        nz = legal ? noise[k] : 0.0;
        have_noise = true;
    } else if (generate_noise) {
        // Dirichlet(alpha) over the legal actions = normalised Gamma(alpha) draws (numpy.random.dirichlet)
        const double gm = legal ? philox_gamma(c.seed, game_id, move, k, c.noise_alpha) : 0.0;
        double sum = gm;
        for (int off = G >> 1; off > 0; off >>= 1) sum += shfl_xor_f64(kWarp, sum, off, G);
        nz = gm / sum;
        have_noise = true;
    }
    if (noise_out && k < A && t.own) noise_out[k] = nz;
    if (k < A && t.own) {
        double p = (double)prior_f32;
        if (legal && have_noise) {
            // prior * (1 - frac) + n * frac       (self_play.py:476)
            p = __dadd_rn(__dmul_rn(p, __dsub_rn(1.0, c.noise_frac)), __dmul_rn(nz, c.noise_frac));
        }
        t.root_prior[k] = legal ? p : 0.0;
        t.visit[k] = 0;
        t.vsum[k] = 0.0;
        t.reward[k] = 0.0f;
        t.prior[k] = legal ? prior_f32 : 0.0f;
        t.expansion[k] = -1;
    }
    t.root_visit = 0;
    t.root_vsum = 0.0;
    t.root_reward = root_reward;
    t.lo = INFINITY;
    t.hi = -INFINITY;
    t.n_expanded = 1;
    t.ties = 0;
    LaneGroup<G>::sync();
}

// ------------------------------------------------------------------------------------------
// Selection: descend from the root until an unexpanded child is reached.
// first_index >= 0: host-supplied pick (index into the tied list) for the all-way tie of the
// first simulation (self_play.py:371-377 with sqrt(0) = 0, see SURVEY.md appendix A.4).
// ------------------------------------------------------------------------------------------
// kPool: the tree lives in the HBM node pool (step-wise pipeline).  Every level is then exactly ONE round trip to
// L2: all fields of this lane's child (and the two table entries of the parent) are requested together, nothing
// is loaded conditionally on a value that has just arrived, and as soon as the child's expansion id is known the
// lines holding ITS children are prefetched into L1, overlapping the score arithmetic of the current level.
template <int G, bool kPool = false>
MZ_DEVINL Leaf tree_select(const TreeConst& c, GameTree& t, int sim, int64_t game_id, int move, int first_index) {
    const int k = LaneGroup<G>::lane();
    const int width = pow2_ceil(c.A);
    int e = 0;
    int n_parent = t.root_visit;
    int depth = 0;
    Leaf leaf;
    bool done = false;                             // the group has reached its leaf: it idles until the warp's last group has
    if (k == 0 && t.own) { t.path[0] = -1; t.path_reward[0] = t.root_reward; }
    do {
        const int base = e * c.A;
        const bool valid = !done && (k < c.A) && (e != 0 || ((t.legal >> k) & 1u));
        double score = -INFINITY;
        int nc = 0, child_exp_k = -1;
        float reward_k = 0.0f;
        if (valid) {
            // one round of independent loads per level: everything this lane's child may need
            nc = t.visit[base + k];
            child_exp_k = t.expansion[base + k];
            const double pr = (e == 0) ? t.root_prior[k] : (double)t.prior[base + k];
            double mv = 0.0, tab_pbc = 0.0, tab_sqrt = 0.0;
            if (kPool) {
                reward_k = t.reward[base + k];
                mv = t.mval[base + k];
                tab_pbc = __ldg(c.pbc + n_parent);
                tab_sqrt = __ldg(c.sqrtn + n_parent);
                if (child_exp_k >= 0) {
                    const int nb = child_exp_k * c.A;
                    prefetch_l1(t.visit + nb); prefetch_l1(t.expansion + nb); prefetch_l1(t.prior + nb);
                    prefetch_l1(t.reward + nb); prefetch_l1(t.mval + nb);
                    prefetch_l1(t.mval + nb + c.A - 1);             // A doubles may straddle a line
                }
            }
            // pb_c = (log(...) + init) * (sqrt(n_p) / (n_c + 1))     self_play.py:384-390
            double pbc;
            if (kPool) {
                pbc = __dmul_rn(tab_pbc, __ddiv_rn(tab_sqrt, (double)(nc + 1)));
            } else if (c.ucb) {
                pbc = __ldg(c.ucb + n_parent * (c.N + 2) + nc);
            } else {
                const double q = __ddiv_rn(c.sqrtn[n_parent], (double)(nc + 1));
                pbc = __dmul_rn(c.pbc[n_parent], q);
            }
            score = __dmul_rn(pbc, pr);
            if (nc > 0) {
                // value_score = normalize(reward + discount * (+/-)mean)  (self_play.py:392-402).  The argument only changes
                // when a backup passes through the child, and the backup evaluates exactly this expression for the
                // min-max statistics: it is stored there (mval) and read back here, which takes an fp64 division and a
                // multiply-add off the per-level critical path without changing a bit.
                if (!kPool) reward_k = t.reward[base + k];
                const double v = value_range_normalize(kPool ? mv : t.mval[base + k], t.lo, t.hi);
                score = __dadd_rn(score, v);
            } else {
                reward_k = 0.0f;                   // (an unvisited child's stored reward is 0 anyway)
                score = __dadd_rn(score, 0.0);     // prior_score + 0
            }
        }
        const double best = group_max_f64<G>(score, width > G ? G : width);
        const unsigned tied = LaneGroup<G>::ballot(valid && score == best);
        const int n_tied = __popc(tied);
        int pick;
        if (done) {
            pick = 0;
        } else if (n_tied <= 1) {
            pick = max(__ffs(tied) - 1, 0);        // n_tied == 0 only for a root without legal actions (rejected by the
                                                   // host; the clamp keeps the slot inside the game's pool regardless)
        } else {
            int idx;
            if (sim == 0 && depth == 0 && first_index >= 0) {
                idx = first_index < n_tied ? first_index : n_tied - 1;
            } else {
                idx = philox_tie_index(c.seed, game_id, move, sim, depth, n_tied);
                if (!(sim == 0 && depth == 0)) t.ties += 1;
            }
            pick = nth_set_bit(tied, idx);
        }
        const int slot = base + pick;
        // the picked child's fields come from the lane that scored it (no second round of loads)
        const int child_exp = LaneGroup<G>::bcast(child_exp_k, pick);
        const int child_visits = LaneGroup<G>::bcast(nc, pick);
        if (!done) {
            depth += 1;
            if (k == pick && t.own) { t.path[depth] = slot; t.path_reward[depth] = reward_k; }
            if (child_exp < 0) {
                leaf.depth = depth;
                leaf.parent_exp = e;
                leaf.action = pick;
                leaf.slot = slot;
                done = true;
            } else {
                n_parent = child_visits;
                e = child_exp;
            }
        }
    } while (LaneGroup<G>::warp_any(!done));
    LaneGroup<G>::sync();
    return leaf;
}

// ------------------------------------------------------------------------------------------
// Multi-level selection (fused FC kernel).  tree_select spends one dependent chain - loads, table lookup, fp64 division,
// shuffle max, ballot, broadcast - per tree level, and with few actions most of the group's lanes idle through it.  Here
// the group scores D levels below the round's start node at once: A + A^2 + ... + A^D <= G lanes, level d (1-based) in
// lanes [off_d, off_d + A^d), off_1 = 0, off_{d+1} = off_d + A^d; lane off_d + j holds the node reached by the base-A
// digits of j (most significant first), i.e. child j % A of level-(d-1) candidate j / A.  Every node's score depends only
// on its own slot, its parent's visit count and lo/hi (constant during a selection), so each lane evaluates exactly
// tree_select's expression for its node; the levels are then resolved in order from two ballots (ties, expanded) with
// tree_select's tie rules at the node's absolute depth, and the next round starts from the last expanded pick.  Same
// scores, same comparisons, same Philox draws: the path is bit-identical to tree_select's.  D = 1 IS tree_select.
// ------------------------------------------------------------------------------------------
constexpr int kMaxSelectLevels = 4;

// levels per round for A actions in a group of G lanes: the largest D with A + A^2 + ... + A^D <= G, capped at what A = 2
// gets (A = 1 would otherwise fill the group)
__host__ __device__ constexpr int select_levels_for(int A, int G) {
    int D = 1, lanes = 0, w = 1;
    for (int d = 1; d <= kMaxSelectLevels; ++d) {
        w *= (A < 2 ? 2 : A);
        if (lanes + w > G) break;
        lanes += w;
        D = d;
    }
    return D;
}

// this lane's place in the layout (fixed for a launch)
struct SelectLanes {
    int D;          // levels per round
    int level;      // 1..D, 0 = idle lane
    int act;        // action of this lane's node (last base-A digit)
    unsigned walk;  // digits 1..level-1 (actions from the round's start node to the parent), 8 bits each
};

template <int G, int kA>
MZ_DEVINL SelectLanes select_lanes(int A_rt, int D) {
    const int A = kA ? kA : A_rt;
    const int k = LaneGroup<G>::lane();
    SelectLanes s{D, 0, 0, 0u};
    int off = 0, w = A, j = 0;
    for (int d = 1; d <= D; ++d) {
        if (k >= off && k < off + w) { s.level = d; j = k - off; }
        off += w;
        w *= A;
    }
    if (s.level > 0) {
        s.act = j % A;
        int q = j / A;
        for (int d = s.level - 1; d >= 1; --d) { s.walk |= (unsigned)(q % A) << (8 * (d - 1)); q /= A; }
    }
    return s;
}

// kMaxD: compile-time bound of sl.D; kA: |A| when fixed at compile time (0 = c.A)
template <int G, int kMaxD, int kA>
MZ_DEVINL Leaf tree_select_lookahead(const TreeConst& c, GameTree& t, const SelectLanes& sl, int sim, int64_t game_id,
                                     int move, int first_index, int& rounds) {
    if (kMaxD <= 1 || sl.D <= 1) {
        const Leaf leaf = tree_select<G>(c, t, sim, game_id, move, first_index);
        rounds = leaf.depth;
        return leaf;
    }
    const int A = kA ? kA : c.A;
    const int D = sl.D;
    const int k = LaneGroup<G>::lane();
    const unsigned seg_mask = (1u << A) - 1u;
    const bool pow2 = (A & (A - 1)) == 0;
    int e = 0;
    int n_parent = t.root_visit;
    int depth = 0;                                 // levels resolved before this round
    Leaf leaf;
    rounds = 0;
    bool done = false;                             // as in tree_select
    if (k == 0 && t.own) { t.path[0] = -1; t.path_reward[0] = t.root_reward; }
    do {
        rounds += done ? 0 : 1;
        // this lane's parent: one dependent (expansion, visit) load per level below the first
        int pe = done ? -1 : e, np = n_parent;
#pragma unroll
        for (int d = 1; d < kMaxD; ++d) {
            if (d < sl.level && pe >= 0) {
                const int s = pe * A + (int)((sl.walk >> (8 * (d - 1))) & 0xffu);
                np = t.visit[s];
                pe = t.expansion[s];
            }
        }
        const bool valid = sl.level > 0 && pe >= 0 && (pe != 0 || ((t.legal >> sl.act) & 1u));
        const int slot = pe * A + sl.act;
        double score = -INFINITY;
        int nc = 0, child_exp_k = -1;
        float reward_k = 0.0f;
        if (valid) {
            // tree_select's score, operation for operation
            nc = t.visit[slot];
            child_exp_k = t.expansion[slot];
            const double pr = (pe == 0) ? t.root_prior[sl.act] : (double)t.prior[slot];
            double pbc;
            if (c.ucb) {
                pbc = __ldg(c.ucb + np * (c.N + 2) + nc);
            } else {
                const double q = __ddiv_rn(c.sqrtn[np], (double)(nc + 1));
                pbc = __dmul_rn(c.pbc[np], q);
            }
            score = __dmul_rn(pbc, pr);
            if (nc > 0) {
                reward_k = t.reward[slot];
                score = __dadd_rn(score, value_range_normalize(t.mval[slot], t.lo, t.hi));
            } else {
                score = __dadd_rn(score, 0.0);
            }
        }
        // maximum over each lane's A siblings, every level at once (exact: no rounding involved)
        double best = score;
        if (pow2) {
            // level offsets are multiples of A: the sibling blocks are aligned
            for (int o = A >> 1; o > 0; o >>= 1) best = fmax(best, shfl_xor_f64(kWarp, best, o, G));
        } else {
            // reduce towards the block's first lane, then broadcast from it
            for (int o = 1; o < A; o <<= 1) {
                const int lo = __shfl_down_sync(kWarp, __double2loint(best), o, G);
                const int hi = __shfl_down_sync(kWarp, __double2hiint(best), o, G);
                if (sl.act + o < A) best = fmax(best, __hiloint2double(hi, lo));
            }
            best = shfl_f64(kWarp, best, k - sl.act, G);
        }
        const unsigned tie_bits = LaneGroup<G>::ballot(valid && score == best);
        const unsigned exp_bits = LaneGroup<G>::ballot(valid && child_exp_k >= 0);
        // resolve the levels in order (uniform over the group)
        int off = 0, w = A, p = 0, last = 0, pick = 0, dl = 0;
        unsigned picked = 0;
        bool hit_leaf = false;
#pragma unroll
        for (int d = 0; d < kMaxD; ++d) {
            if (d < D && !hit_leaf && !done) {
                const int seg = off + p * A;
                const unsigned tied = (tie_bits >> seg) & seg_mask;
                const int n_tied = __popc(tied);
                const int dd = depth + d;          // absolute depth of the parent
                if (n_tied <= 1) {
                    pick = max(__ffs(tied) - 1, 0);
                } else {
                    int idx;
                    if (sim == 0 && dd == 0 && first_index >= 0) {
                        idx = first_index < n_tied ? first_index : n_tied - 1;
                    } else {
                        idx = philox_tie_index(c.seed, game_id, move, sim, dd, n_tied);
                        if (!(sim == 0 && dd == 0)) t.ties += 1;
                    }
                    pick = nth_set_bit(tied, idx);
                }
                last = seg + pick;
                picked |= 1u << last;
                dl = d + 1;
                hit_leaf = ((exp_bits >> last) & 1u) == 0;
                off += w;
                w *= A;
                p = p * A + pick;
            }
        }
        if (((picked >> k) & 1u) && t.own) { t.path[depth + sl.level] = slot; t.path_reward[depth + sl.level] = reward_k; }
        // (picked == 0 once done) the leaf's parent, or the next round's start node and its visit count
        const int next = LaneGroup<G>::bcast(hit_leaf ? pe : child_exp_k, last);
        const int next_visits = LaneGroup<G>::bcast(nc, last);
        if (hit_leaf) {
            leaf.depth = depth + dl;
            leaf.parent_exp = next;
            leaf.action = pick;
            leaf.slot = next * A + pick;
            done = true;
        } else if (!done) {
            e = next;
            n_parent = next_visits;
            depth += D;
        }
    } while (LaneGroup<G>::warp_any(!done));
    LaneGroup<G>::sync();
    return leaf;
}

// ------------------------------------------------------------------------------------------
// Expansion of the selected leaf with the network outputs (self_play.py:345-351, 451-465).
// prior_f32: this lane's fp32 softmax prior (lane k <-> action k).
// ------------------------------------------------------------------------------------------
template <int G, int kA = 0>
MZ_DEVINL int tree_expand(const TreeConst& c, GameTree& t, const Leaf& leaf, float reward, float prior_f32) {
    const int A = kA ? kA : c.A;
    const int k = LaneGroup<G>::lane();
    const int e = t.n_expanded;
    if (k == 0 && t.own) {
        t.expansion[leaf.slot] = e;
        t.reward[leaf.slot] = reward;
        t.path_reward[leaf.depth] = reward;
    }
    if (k < A && t.own) {
        const int s = e * A + k;
        t.visit[s] = 0;
        t.vsum[s] = 0.0;
        t.reward[s] = 0.0f;
        t.prior[s] = prior_f32;
        t.expansion[s] = -1;
    }
    t.n_expanded = e + 1;
    LaneGroup<G>::sync();
    return e;
}

// ------------------------------------------------------------------------------------------
// Backup along path[0..depth] (self_play.py:406-430).  The discounted value recurrence is a
// serial chain (2 fp64 ops per level, run redundantly by every lane); the per-node updates
// (value_sum, visit, running min/max) are independent: lane j updates node j, all at once, after
// the recurrence handed every lane the value its node saw.
// ------------------------------------------------------------------------------------------
// RN(s / n), n = a visit count + 1: div_by_count when kRcp, else the IEEE division
template <bool kRcp>
MZ_DEVINL double mean_of(double s, int n) {
    if constexpr (kRcp) return div_by_count(s, n, __drcp_rn((double)n));
    else return __ddiv_rn(s, (double)n);
}

// kP: number of players when fixed at compile time (0 = c.P).
// kRcp: the means divide through div_by_count.  After a shuffled recurrence every lane then reads its node's sum and count
// and takes RN(1 / count) BEFORE the recurrence (that work overlaps the serial chain instead of following it), evaluates
// the update (a lane without a node on slot 0, with a numerator of 1) and stores it predicated: three dependent fp64 steps
// behind the recurrence instead of a division, and no divergent owner block.
template <int G, int kP = 0, bool kRcp = false>
MZ_DEVINL void tree_backup(const TreeConst& c, GameTree& t, const Leaf& leaf, float leaf_value) {
    const int P = kP ? kP : c.P;
    const int k = LaneGroup<G>::lane();
    const int L = leaf.depth;                         // path indices 0..L
    double lo = INFINITY, hi = -INFINITY;
    double v = (double)leaf_value;                    // value seen by node j, starting at j = L
    double root_vsum = t.root_vsum;
    // lane j holds (slot, reward) of path node j when the path fits in the group: the serial recurrence
    // then runs on shuffles instead of a dependent chain of loads.  Its shuffles are collectives, so the choice and the trip
    // count follow the deepest path of the warp (Lw); the shallower groups' steps j > L change nothing.
    const int Lw = G < 32 ? (int)__reduce_max_sync(kWarp, (unsigned)L) : L;
    const bool packed = (Lw < G);
    int my_slot = -1;
    float my_reward = 0.0f;
    if (packed && k <= L) { my_slot = t.path[k]; my_reward = t.path_reward[k]; }
    if (packed) {
        // The recurrence runs on shuffles and every lane keeps the value its own node saw; the node updates then happen
        // ONCE, all lanes in parallel (a divergent owner block inside the loop would be issued L + 1 times, one lane each).
        const bool mine = kRcp && k <= L && t.own;  // (kRcp) this lane updates a node
        const int sl = (mine && k > 0) ? my_slot : 0;
        double old_sum = 0.0, y = 1.0;
        int n = 1;
        if constexpr (kRcp) {
            old_sum = k == 0 ? t.root_vsum : t.vsum[sl];
            n = mine ? (k == 0 ? t.root_visit : t.visit[sl]) + 1 : 1;
            y = __drcp_rn((double)n);
        }
        double myv = 0.0;
        for (int j = Lw; j >= 0; --j) {
            const double r = (double)LaneGroup<G>::bcast(my_reward, j);
            const bool same = (P == 1) || (((L - j) & 1) == 0);
            if (j == k) myv = v;
            const double rr = (P == 1) ? r : (same ? -r : r);
            const double vn = __dadd_rn(rr, __dmul_rn(c.discount, v));
            v = j <= L ? vn : v;
        }
        if constexpr (kRcp) {
            const bool same = (P == 1) || (((L - k) & 1) == 0);
            const double add = same ? myv : -myv;
            const double s = __dadd_rn(old_sum, add);
            const double q = div_by_count(mine ? s : 1.0, n, y);
            const double m = __dadd_rn((double)my_reward, __dmul_rn(c.discount, (P == 1) ? q : -q));
            if (mine && k > 0) { t.vsum[sl] = s; t.visit[sl] = n; t.mval[sl] = m; }   // mval: what the next selection normalises
            if (mine && k == 0) root_vsum = s;
            lo = mine ? m : lo;
            hi = mine ? m : hi;
        } else if (k <= L && t.own) {
            const bool same = (P == 1) || (((L - k) & 1) == 0);
            const double add = same ? myv : -myv;
            double q;
            if (k == 0) {
                root_vsum = __dadd_rn(t.root_vsum, add);
                q = __ddiv_rn(root_vsum, (double)(t.root_visit + 1));
            } else {
                const double s = __dadd_rn(t.vsum[my_slot], add);
                const int n = t.visit[my_slot] + 1;
                t.vsum[my_slot] = s;
                t.visit[my_slot] = n;
                q = __ddiv_rn(s, (double)n);
            }
            const double m = __dadd_rn((double)my_reward, __dmul_rn(c.discount, (P == 1) ? q : -q));
            if (k > 0) t.mval[my_slot] = m;           // what the next selection will normalise for this child
            lo = m;
            hi = m;
        }
    } else {
    for (int j = L; j >= 0; --j) {                    // (no collective in this loop: its trip count may differ per group)
        const int slot = t.path[j];
        const float rf = t.path_reward[j];
        const double r = (double)rf;
        // node.to_play == to_play  <=>  (L - j) even (players alternate every level)
        const bool same = (P == 1) || (((L - j) & 1) == 0);
        if ((j % G) == k && t.own) {
            const double add = same ? v : -v;
            double q;
            if (j == 0) {
                root_vsum = __dadd_rn(t.root_vsum, add);
                q = mean_of<kRcp>(root_vsum, t.root_visit + 1);
            } else {
                const double s = __dadd_rn(t.vsum[slot], add);
                const int n = t.visit[slot] + 1;
                t.vsum[slot] = s;
                t.visit[slot] = n;
                q = mean_of<kRcp>(s, n);
            }
            const double m = __dadd_rn(r, __dmul_rn(c.discount, (P == 1) ? q : -q));
            if (j > 0) t.mval[slot] = m;           // what the next selection will normalise for this child
            lo = fmin(lo, m);
            hi = fmax(hi, m);
        }
        // value = (same ? -reward : reward) + discount * value     (P == 2)
        // value = reward + discount * value                        (P == 1)
        const double rr = (P == 1) ? r : (same ? -r : r);
        v = __dadd_rn(rr, __dmul_rn(c.discount, v));
    }
    }
    // only lanes 0..L hold candidates: reduce over the smallest power of two covering the warp's deepest path (the others
    // hold the neutral +-inf), then broadcast lane 0's result (lanes beyond the reduced width hold partial values)
    const int width = (Lw + 1 >= G) ? G : pow2_ceil(Lw + 1);
    const unsigned gm = kWarp;
    if (width >= 2) {
        // minimum and maximum in ONE butterfly: after the first exchange the lower half of the `width` lanes carries minimum
        // candidates and the upper half maximum candidates (each lane sends the one it does not keep), the remaining steps
        // stay inside the halves; lane 0 ends with the minimum, lane width/2 with the maximum (exact: no rounding involved)
        const int half = width >> 1;
        const bool up = (k & half) != 0;
        const double got = shfl_xor_f64(gm, up ? lo : hi, half, G);
        double val = up ? fmax(hi, got) : fmin(lo, got);
        for (int off = half >> 1; off > 0; off >>= 1) {
            const double r = shfl_xor_f64(gm, val, off, G);
            val = up ? fmax(val, r) : fmin(val, r);
        }
        lo = shfl_f64(gm, val, 0, G);
        hi = shfl_f64(gm, val, half, G);
    } else {
        lo = shfl_f64(gm, lo, 0, G);
        hi = shfl_f64(gm, hi, 0, G);
    }
    root_vsum = shfl_f64(gm, root_vsum, 0, G);
    t.root_vsum = root_vsum;
    t.root_visit += 1;
    t.lo = fmin(t.lo, lo);
    t.hi = fmax(t.hi, hi);
    LaneGroup<G>::sync();
}

}  // namespace mz
