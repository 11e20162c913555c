// Step-wise search pipeline over the HBM node pool + the residual-network interface.
#pragma once
#include <string>

#include "kernels.h"

namespace mz {

// One mz_search call after host staging: every pointer is a device pointer.
struct SearchCall {
    int n;
    const float* obs;
    const uint8_t* legal_mask;
    const int32_t* to_play;
    int add_noise;
    const double* noise;
    const int32_t* first_index;
    const int64_t* game_id;
    const int32_t* move_index;
    int32_t* visit_counts;
    double* root_value;
    float* root_predicted_value;
    int32_t* max_tree_depth;
    int32_t* tie_count;
    double* root_priors;
    double* value_range;
    DevTeacher teacher;
    DevTrace trace;
    bool keep_tree;
    size_t out_bytes;
    int continue_from;             // > 0: MZ_FLAG_CONTINUE, the pool already holds this many expansions of every game
    // Partitioned replay (abi.cu): the games [g0, g0 + n) of the batch, every array still addressed by the GLOBAL game
    // index, and only some phases of the search.  g0 = 0, phases = kPhaseAll is the plain whole-batch call.
    int g0;
    int phases;
};
constexpr int kPhaseRoot = 1, kPhaseSims = 2, kPhaseAll = 0;      // 0 = both (so a zero-initialised call is a whole search)

// One batched network call. Plain mode: sample g reads in[g*in_elems...] and writes hidden[g*H...].
// Pool mode (gather_parent != nullptr): sample g reads pool_hidden[(g*pool_stride + gather_parent[g])*H...]
// and writes its new state to pool_hidden[(g*pool_stride + out_slot)*H...].
struct InferCall {
    int n, recurrent;
    int g0;                        // first game of the call: every per-game array is addressed by g0 + local index
    const float* in;
    const int32_t* action;
    const int32_t* gather_parent;
    float* pool_hidden;
    int pool_stride, out_slot;
    float *value_logits, *reward_logits, *policy_logits, *hidden, *value, *reward;
};

// One launch of the step-wise tree kernel (tree_kernels.cu).
struct TreeStepArgs {
    int n, N, A, P;
    int g0;                        // games [g0, g0 + n), arrays addressed by the global index
    int sim;                       // simulation selected by this launch (do_select); do_update handles sim-1
    int do_root, do_update, do_select, do_final;
    double discount, noise_frac, noise_alpha;
    uint64_t seed;
    const double* pbc;
    const double* sqrtn;
    const double* ucb;
    NodePool pool;
    const uint8_t* legal_mask;
    const double* noise;
    int add_noise;
    const int32_t* first_index;
    const int64_t* game_id;
    const int32_t* move_index;
    // outputs of the network (or teacher table) for the node being expanded
    const float* net_value;        // [g*value_stride]
    const float* net_reward;       // [g*value_stride]; nullptr at the root = log(one-hot centre)
    const float* net_policy;       // [g*policy_stride + k] logits, or priors if policy_is_prior
    int value_stride, policy_stride, policy_is_prior;
    // final outputs
    int32_t* visit_counts; double* root_value; float* root_predicted_value; int32_t* max_tree_depth;
    int32_t* tie_count; double* root_priors; double* value_range;
    DevTrace trace;
};
cudaError_t launch_tree_step(const TreeStepArgs& a, cudaStream_t stream);
cudaError_t launch_tree_step_wide(const TreeStepArgs& a, cudaStream_t stream);      // 32 < |A| <= 256 (tree_wide.cu)
cudaError_t launch_tree_adopt_root(const TreeStepArgs& a, cudaStream_t stream);     // MZ_FLAG_CONTINUE: adopt the imported tree

// How a residual net runs its towers, chosen once at resnet_create (resnet_use_strict moves a guarded route to CudaCore).
//   CudaCore  fp32 conv3x3_kernel / fused small towers, dense NCHW states
//   TcF16     64-channel tensor-core towers on fp16 operands (MZ_TC_MODE=fp16), P64C8 board states
//   TcX3      64-channel tensor-core towers on split operands (default where the board allows), x_h | x_l board states
//   Wide      128-channel x3 tensor-core towers, one CTA per board (MZ_TC_WIDE=1), dense states
//   WidePair  the same, each board split across a CTA pair (MZ_TC_WIDE=2), dense states
//   Wide256   256-channel x3 tensor-core towers, output channels split across a CTA pair (MZ_TC_WIDE=3), dense states
enum class TowerRoute { CudaCore, TcF16, TcX3, Wide, WidePair, Wide256 };

struct ResNetDevice;
ResNetDevice* resnet_create(const MzNetDesc& net, int max_batch, int sm_count, std::string* err);
void resnet_destroy(ResNetDevice* r);
int resnet_load_weights(ResNetDevice* r, const MzTensor* tensors, int n, std::string* err);
int resnet_inference(ResNetDevice* r, const InferCall& c, cudaStream_t stream, int64_t* launches, std::string* err);
int resnet_debug_conv(int n, int cin, int cout, int H, int W, int stride, const float* x, const float* w_oihw, const float* bias,
                      const float* residual, int relu, int use_tc, float* out, int sm_count, std::string* err);
int resnet_debug_downsample(int n, int in, int C, int H, int W, const float* x, const float* w, const float* bias, float* out,
                            float* stages, int sm_count, std::string* err);
bool resnet_conv_plan(int n, int cin, int cout, int H, int W, int stride, int64_t* plan, std::string* err);   // host only
const char* resnet_numerics(const ResNetDevice* r);                  // arithmetic of the residual towers (bench.py dtype)
int resnet_take_saturations(ResNetDevice* r, cudaStream_t stream);   // x3 range guard (synchronises)
bool resnet_can_partition(const ResNetDevice* r);
// games per range of the partitioned replay (the last range may hold fewer): a multiple of 8
inline int partition_games(int n, int parts) { return ((n + parts - 1) / parts + 7) & ~7; }
// Debug / parity entry behind mz_debug_conv_tower (route TcF16 / TcX3, C = 64), mz_debug_small_tower (CudaCore: the fused
// CUDA-core tower), mz_debug_wide_tower (Wide, C = 128), mz_debug_wide_pair_tower (WidePair) and mz_debug_wide256_tower
// (Wide256, C = 256): one tower of one call site of the network on host NCHW data (see include/mzb200.h).  `in_channels`
// is the planes the representation stem reads (CudaCore only; C otherwise); `launches`, `saturated` and `plan` (plan[6]
// fused, plan[9] wide, plan[10] Wide256) may be null; `force_boards` (Wide256 only) forces the boards per CTA pair.
int resnet_debug_tower(TowerRoute route, int n, int in_channels, int C, int H, int W, int blocks, int site, int parts, int A,
                       const float* x, const float* w, const float* bias, const int32_t* action, const int32_t* parent,
                       int pool_stride, float* out, int64_t* launches, int32_t* saturated, int64_t* plan, int sm_count,
                       std::string* err, int force_boards = 0);
// Host-only plan of the fused CUDA-core tower (plan[6], see include/mzb200.h, mz_debug_small_tower_plan)
bool resnet_small_tower_plan(int n, int in_channels, int C, int H, int W, int blocks, bool stem, int sm_count, int64_t* plan,
                             std::string* err);
// Host-only plan of the wide 128-channel tower (plan[9], see include/mzb200.h, mz_debug_wide_tower_plan; with `pair`
// mz_debug_wide_pair_tower_plan), one CTA (a CTA pair) per board
bool resnet_wide_tower_plan(int n, int C, int H, int W, int blocks, bool stem, int sm_count, int64_t* plan, std::string* err,
                            bool pair = false);
// Host-only plan of the 256-channel tower (plan[10], see include/mzb200.h, mz_debug_wide256_tower_plan)
bool resnet_wide256_tower_plan(int n, int C, int H, int W, int blocks, bool stem, int sm_count, int force_boards, int64_t* plan,
                               std::string* err);
// Host-only plan of one heads call (plan[5], see include/mzb200.h, mz_debug_heads_plan) and the debug / parity entry behind
// mz_debug_heads: the heads of one call site of resnet_inference on host NCHW data, in any of the three state layouts
bool resnet_heads_plan(int n, int g0, int C, int H, int W, int site, int layout, int route, const int32_t* shapes, int sm_count,
                       int64_t* plan, std::string* err);
int resnet_debug_heads(int n, int C, int H, int W, int site, int layout, int route, int parts, const int32_t* shapes,
                       const MzTensor* tensors, int n_tensors, const float* x, int pool_stride, int out_slot, float* logits0,
                       float* logits1, float* scalar, float* rescaled, float* pool, float* state, int64_t* plan, int sm_count,
                       std::string* err);
// fused search of small residual networks: all simulations in one launch (small_search.cu); MZ_SMALL_SEARCH=0 / 1 switches it off / on
bool resnet_small_search_supported(ResNetDevice* r, const InferCall& first_recurrent, const TreeStepArgs& tree, int n_sims);
int resnet_small_search(ResNetDevice* r, const InferCall& first_recurrent, const TreeStepArgs& tree, int n_sims, cudaStream_t stream,
                        int64_t* launches, std::string* err);
bool resnet_uses_tensor_cores(const ResNetDevice* r);   // the 64-channel tensor-core towers (TcF16 / TcX3)
void resnet_use_strict(ResNetDevice* r);                // fp32 CUDA-core towers from now on (the range guard fired)
int resnet_state_elems(const ResNetDevice* r);        // floats per stored hidden state in the pool
int resnet_states_to_nchw(ResNetDevice* r, const float* states, int count, float* out, cudaStream_t stream);

cudaError_t launch_fc_inference_pool(const FcNet& net, const float* blob, const InferCall& c, int group, int sm_count, size_t smem_cap,
                                     cudaStream_t stream);

int resnet_states_from_nchw(ResNetDevice* r, const float* dense, int count, float* states, cudaStream_t stream);

int run_stepwise_search(const MzNetDesc& net, const MzSearchDesc& search, int pool_n, const NodePool& pool, const double* d_pbc,
                        const double* d_sqrt, const double* d_ucb, const FcNet& fc, const float* d_fc_blob, ResNetDevice* res,
                        const SearchCall& call, int fc_group, int sm_count, size_t smem_cap, cudaStream_t stream, int64_t* launches,
                        std::string* err);

}  // namespace mz
