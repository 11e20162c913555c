// Internal interface between the host side of the library (abi.cu) and the kernel files.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/mzb200.h"
#include "fc_net.cuh"

namespace mz {

constexpr int kFcThreads = 128;      // fc_inference_kernel block
// Upper bound of the fused search kernel's block.  Two such CTAs per SM at the 128 registers per thread that
// __launch_bounds__(kFcMaxThreads, 2) caps the kernel at fill the 64K-register file exactly (fc_search_plan).
constexpr int kFcMaxThreads = 256;

// HBM node pool, game-major: game g owns slots [g*(N+1)*A, (g+1)*(N+1)*A).
struct NodePool {
    int* visit;            // [B, (N+1)*A]
    double* vsum;          // [B, (N+1)*A]
    double* mval;          // [B, (N+1)*A] cached reward + discount * (+/-)mean of every visited child (tree.cuh)
    float* reward;         // [B, (N+1)*A]
    float* prior;          // [B, (N+1)*A]
    int* expansion;        // [B, (N+1)*A]
    double* root_prior;    // [B, A]
    float* hidden;         // [B, N+1, hidden_elems]
    int* root_visit;       // [B]
    double* root_vsum;     // [B]
    float* root_reward;    // [B]
    double* range;         // [B, 2]
    int* n_expanded;       // [B]
    int* ties;             // [B]
    int* max_depth;        // [B]
    unsigned* legal;       // [B]
    int* path;             // [B, N+2]
    float* path_reward;    // [B, N+2]
    // leaf of the simulation in flight
    int* leaf_depth;       // [B]
    int* leaf_parent;      // [B]
    int* leaf_action;      // [B]
    int* leaf_slot;        // [B]
    // network outputs of the evaluation in flight (step-wise pipeline)
    float* net_value;      // [B]
    float* net_reward;     // [B]
    float* net_policy;     // [B, A]
};

struct DevTeacher { const float *root_value, *root_reward, *root_priors, *value, *reward, *priors; };
struct DevTrace {
    int max_depth;
    int* depth; uint8_t* actions; float *value, *reward, *priors, *root_priors_raw, *root_reward;
    double* noise;         // [n, A] Dirichlet noise actually mixed in (host-given or device-drawn)
};

struct FcSearchArgs {
    int n_games, N, A, P;
    int threads;           // block size of the launch (multiple of 32), 0 = the one fc_search_plan picks
    int select_levels;     // tree levels per selection round (set by launch_fc_search)
    double discount, noise_frac, noise_alpha;
    uint64_t seed;
    const double* pbc;
    const double* sqrtn;
    const double* ucb;
    FcNet net;
    const float* blob;
    // inputs (device)
    const float* obs;
    const uint8_t* legal_mask;
    const int32_t* to_play;
    int add_noise;
    const double* noise;
    const int32_t* first_index;
    const int64_t* game_id;
    const int32_t* move_index;
    // outputs (device)
    int32_t* visit_counts;
    double* root_value;
    float* root_predicted_value;
    int32_t* max_tree_depth;
    int32_t* tie_count;
    double* root_priors;
    double* value_range;
    DevTeacher teacher;
    DevTrace trace;
    NodePool pool;         // pool.visit == nullptr unless MZ_FLAG_KEEP_TREE
};

struct FcInferArgs {
    int n, recurrent;
    FcNet net;
    const float* blob;
    const float* in;          // obs [n, obs_elems] (initial) or hidden [n, E] (recurrent)
    const int32_t* action;    // [n] (recurrent)
    // pool mode: sample g reads pool_hidden[(g*pool_stride + gather_parent[g])*E ...] and writes its
    // new state to pool_hidden[(g*pool_stride + out_slot)*E ...]
    const int32_t* gather_parent;
    float* pool_hidden;
    int pool_stride, out_slot;
    float *value_logits, *reward_logits, *policy_logits, *hidden, *value, *reward;
};
// smem_cap: the device's shared memory per block (opt-in), which the CTA is sized to (fc_infer_plan)
cudaError_t launch_fc_inference(const FcInferArgs& a, int group, int sm_count, size_t smem_cap, cudaStream_t stream);

// Launch of fc_inference_kernel<G> over n samples: `threads` per CTA of `groups` samples, `grid` CTAs (at most 8 per SM; the
// CTAs stride over the rest), `smem` bytes: the weight blob, then 4 maxw + 4 floats of scratch per group.
struct FcInferPlan { int threads, groups, grid; size_t smem; };
inline size_t fc_infer_smem(int blob_floats, int maxw, int groups) {
    return (((size_t)blob_floats + 3) & ~(size_t)3) * 4 + (size_t)groups * (4 * (size_t)maxw + 4) * 4;
}
// False when not even one warp's groups fit next to the blob in smem_cap bytes (mz_load_weights refuses such a net).
bool fc_infer_plan(int blob_floats, int maxw, int G, int n, int sm_count, size_t smem_cap, FcInferPlan* plan);

// mz_debug_fc_net: one network call of the search (routes MZ_FC_SEARCH_*) for each of n samples.  Output rows of n x E
// (raw: the next or initial state before the rescale; hidden: after it), n x F / n x A logits, n x A priors and n scalars;
// a null pointer is not written.
struct FcDebugArgs {
    int n, route;
    bool force_split;
    FcNet net;
    const float* blob;
    const float* in;            // obs [n, obs_elems] (root) or parent states [n, E] (simulation)
    const int32_t* action;      // [n] (simulation)
    float *raw, *hidden, *reward_logits, *value_logits, *policy_logits, *prior, *value, *reward;
};
// plan[5] = {path (MZ_FC_PATH_*), G, threads, grid, smem} of a route, or false and the reason
bool fc_debug_plan(const FcNet& net, int G, int route, bool force_split, int n, int sm_count, size_t smem_cap, int64_t* plan,
                   std::string* err);
cudaError_t launch_fc_debug_net(const FcDebugArgs& a, int G, const int64_t* plan, cudaStream_t stream);

struct FcLaunchInfo { int grid, block, ctas_per_sm, group; size_t smem; };

// Launch shape of the fused search: `threads` per CTA of `groups` games and `smem` bytes, `ctas_per_sm` resident per SM,
// `slots` games resident on the GPU at once, `passes` = ceil(n_games / slots) chains of the persistent loop.
struct FcPlan { int threads, groups, ctas_per_sm, slots, passes; size_t smem; };

// Host arithmetic only.  Over CTAs of 64, 128 and 256 threads (or `threads` alone when it is not 0), the one whose resident
// CTAs - limited by shared memory (smem_per_sm, less smem_reserve per CTA), registers (regs per thread) and threads per SM -
// run n_games in the fewest passes, and the smallest of those.  False when one game's tree does not fit a CTA (smem_cap).
bool fc_search_plan(int N, int A, int E, int maxw, int blob_floats, int G, bool teacher, int n_games, int sm_count,
                    size_t smem_per_sm, size_t smem_reserve, size_t smem_cap, int regs, int threads, FcPlan* plan);

// What decides a fused launch besides the handle's fixed network and tree shape: the games, the lanes per game, a fixed
// CTA size (0 = planned), teacher forcing and the two A/B switches (MZ_FC_GENERIC, MZ_FC_SELECT_LEVELS).
struct FcPreparedKey {
    int n_games, group, threads;
    bool teacher, generic, one_level;
    bool operator==(const FcPreparedKey& o) const {
        return n_games == o.n_games && group == o.group && threads == o.threads && teacher == o.teacher &&
               generic == o.generic && one_level == o.one_level;
    }
};

// The launch made for `key`: instantiation, selection levels and shape.  A search with the same key only copies its
// pointers into the arguments and launches.
struct FcPrepared {
    bool valid = false;
    FcPreparedKey key{};
    int select_levels = 1;
    bool fixed_shape = false;      // the instantiation with the unrolled network of FcFixedShape
    cudaError_t (*launch)(const FcSearchArgs&, const FcLaunchInfo&, cudaStream_t) = nullptr;
    FcLaunchInfo info{};
};

// The device limits the plan is made against, and what a handle has set up for the fused search kernel so far: each
// instantiation gets its attributes set and its register count read once, each (instantiation, block, shared memory)
// its occupancy confirmed once, and the launch of the last key is kept, so that later searches go straight to the launch.
struct FcLaunchState {
    size_t smem_per_sm = 0, smem_reserve = 0, smem_cap = 0;
    struct Kernel { const void* fn; int regs; };
    struct Shape { const void* fn; int threads; size_t smem; int ctas_per_sm; };
    std::vector<Kernel> kernels;
    std::vector<Shape> shapes;
    FcPrepared prepared;           // invalidated when the weights load (the network descriptors are replaced)
    bool launched = false;         // last: the handle's last fused launch (mz_fc_last_launch)
    FcLaunchInfo last{};
};

cudaError_t launch_fc_search(const FcSearchArgs& a, int group, bool teacher, int sm_count, FcLaunchState* state,
                             cudaStream_t stream);

}  // namespace mz
