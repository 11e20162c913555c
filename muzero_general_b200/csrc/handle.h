// The library handle and the helpers shared by the entry-point files (abi.cu, selfplay.cu, reanalyse.cu).
#pragma once
#include <time.h>

#include <map>
#include <string>
#include <vector>

#include "kernels.h"
#include "pipeline.h"
#include "ktimer.h"

struct MzSelfPlay;                     // device-resident self-play state (selfplay.cu)
struct MzReanalyse;                    // Reanalyse's staging buffers and copy stream (reanalyse.cu)
struct MzUserEnvCache;                 // compiled user environments of mz_selfplay_begin_user (user_env.cu)
using namespace mz;

struct MzHandle {
    MzNetDesc net;
    MzSearchDesc search;
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::string err;
    int64_t launches = 0;
    double last_ms = 0.0;
    // tables
    double* d_pbc = nullptr;
    double* d_sqrt = nullptr;
    double* d_ucb = nullptr;           // optional host-evaluated exploration-factor table
    // fully-connected weights
    FcNet fc{};
    float* d_fc_blob = nullptr;
    bool weights_loaded = false;
    int fc_group = 16;
    int fc_threads = 0;                // CTA size of the fused search, 0 = planned per launch (MZ_FC_THREADS overrides)
    FcLaunchState fc_launch;
    // residual weights + workspace
    ResNetDevice* res = nullptr;
    // pool
    NodePool pool{};
    int64_t hidden_elems = 0, obs_elems = 0;
    int64_t pool_state_elems = 0;      // floats per hidden state as stored in the pool (layout dependent)
    // IO arenas
    unsigned char* d_in = nullptr;
    unsigned char* d_out = nullptr;
    unsigned char* h_in = nullptr;
    unsigned char* h_out = nullptr;
    size_t in_cap = 0, out_cap = 0;
    // CUDA graphs of the step-wise pipeline, one per argument set (callers that rotate a few input buffers - double
    // buffering, bench.py's four batches - keep replaying): a set seen twice is captured, the least recently used of
    // kMaxGraphs entries makes room
    struct SearchGraph {
        uint64_t key = 0;
        int seen = 0;
        cudaGraphExec_t exec = nullptr;
        int64_t launches = 0;
        int parts = 1;
        uint64_t used = 0;             // tick of the last use
    };
    static constexpr int kMaxGraphs = 8;
    std::vector<SearchGraph> graphs;
    uint64_t graph_tick = 0;
    // partitioned replay: the simulations of disjoint game ranges run as parallel branches of the graph (abi.cu)
    static constexpr int kMaxParts = 4;
    cudaStream_t part_stream[kMaxParts] = {nullptr, nullptr, nullptr, nullptr};     // [0] unused (= stream)
    cudaEvent_t part_fork = nullptr, part_join[kMaxParts] = {nullptr, nullptr, nullptr, nullptr};
    int graph_parts = 1;               // branches of the graph replayed last (mz_graph_partitions)
    // lazily allocated debug buffers
    std::vector<void*> debug_allocs;
    std::map<std::string, std::pair<void*, size_t>> named;
    MzSelfPlay* sp = nullptr;          // mz_selfplay_begin
    MzReanalyse* ra = nullptr;         // mz_reanalyse_values, on first use
    MzUserEnvCache* user_env = nullptr;   // mz_selfplay_begin_user's modules by source, on first use
    int64_t user_env_compiles = 0;     // NVRTC compiles made for this handle (mz_debug_user_env_compiles)
    int pool_n = 0;                    // layout "N" of the node pool and tables: num_simulations + extra_expansions
    int imported_expansions = 0;       // expansions of the tree mz_import_tree seeded last (MZ_FLAG_CONTINUE)
    int range_fallbacks = 0;           // times the x3 range guard switched this handle to the fp32 towers (0 or 1)
    // the search mz_search_device enqueued and mz_search_device_wait has not waited for yet
    mz::SearchCall device_call{};
    bool device_pending = false;
    // CLOCK_MONOTONIC ns of the last search call: entry, search enqueued, stream synchronised, return
    // (mz_debug_host_split; scripts/search_host_split.py)
    int64_t host_ns[4] = {0, 0, 0, 0};
};

static inline int64_t mz_host_ns() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (int64_t)ts.tv_sec * 1000000000 + ts.tv_nsec;
}

int mz_fail(MzHandle* h, int code, const std::string& msg);
static inline int fail(MzHandle* h, int code, const std::string& msg) { return mz_fail(h, code, msg); }

#define MZ_CUDA(h, expr)                                                                          \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            return fail(h, MZ_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));          \
    } while (0)


// One batched search on device buffers, enqueued on h->stream without synchronising: the fused FC kernel or the
// step-wise pipeline (eager for the first two calls with a given argument set, then a CUDA-graph replay).
int mz_dispatch_search(MzHandle* h, const mz::SearchCall& call, bool teacher, bool trace, int flags);
// One batched network call (mz_initial_inference / mz_recurrent_inference's): the FC kernel or resnet_inference, enqueued
// on h->stream.  mz_network_guard then synchronises; when the x3 towers' range guard fired it switches the handle to the
// fp32 towers and enqueues the call again.
int mz_network_enqueue(MzHandle* h, const mz::InferCall& c);
int mz_network_guard(MzHandle* h, const mz::InferCall& c);
void mz_reanalyse_destroy(MzHandle* h);
void mz_selfplay_destroy(MzHandle* h);
// The wrapper kernels of a user environment (user_env.cuh) compiled from `source`, from the handle's cache or by NVRTC;
// expert is nullptr for a source without MZ_ENV_EXPERT (user_env_expert.cuh).
struct MzUserEnvKernels {
    cudaKernel_t reset = nullptr, step = nullptr, expert = nullptr;
};
int mz_user_env_kernels(MzHandle* h, const char* source, MzUserEnvKernels* out);
void mz_user_env_destroy(MzHandle* h);
void mz_switch_to_strict(MzHandle* h);
void mz_drop_graphs(MzHandle* h);             // captured graphs refer to buffers or kernels that are about to change
