// Step-wise tree kernels over the HBM node pool (game-major SoA, see kernels.h / tree.cuh).
//
// One launch per simulation performs, for every game of the batch,
//   [root expansion]  ->  [expand + backup of the previous simulation's leaf]  ->
//   [selection of the next leaf]  ->  [final read-out]
// (phases enabled by flags), so that a search of N simulations is N+1 tree launches with the
// batched network evaluation in between.  A group of G >= |A| lanes owns one game: the A child
// slots of a node are read with one coalesced access per array, scores are reduced with
// shuffles, and the per-node backup updates are spread over the lanes (tree.cuh).
#include "kernels.h"
#include "pipeline.h"
#include "tree.cuh"
#include "tree_step.cuh"
#include "launch.h"

#include <stdlib.h>

namespace mz {

// kLatency: few games in flight (the launch is bound by the chain of dependent round trips to L2, not by
// throughput): selection uses the single-round-trip + L1-prefetch variant of tree_select (tree.cuh).
template <int G, bool kLatency>
__global__ void __launch_bounds__(128) tree_step_kernel(const __grid_constant__ TreeStepArgs a) {
    pdl_launch_dependents();
    pdl_wait();                                   // everything below reads what the network kernels just wrote
    // a warp with a game runs whole: a group past the last game replays the last one (in this warp) and stores nothing
    const int first = (blockIdx.x * blockDim.x + (threadIdx.x & ~31u)) / G;
    if (first >= a.n) return;
    const int local = (blockIdx.x * blockDim.x + threadIdx.x) / G;
    const bool own = local < a.n;
    tree_step_game<G, kLatency>(a, a.g0 + (own ? local : a.n - 1), own, a.sim, a.do_root, a.do_update, a.do_select,
                                a.do_final);   // arrays are addressed by the global game index
}

// override_root_with (self_play.py:275-277, 310-314): the tree mz_import_tree put into the pool becomes the root of a new
// search - fresh MinMaxStats, tie / depth counters reset, and the exploration noise mixed into the priors the root's
// children already have (self_play.py:467-476).  Its own kernel (one game per lane group, launched once per continued
// search) so that the per-simulation kernel keeps its register budget.
template <int G>
__global__ void __launch_bounds__(128) tree_adopt_root_kernel(const __grid_constant__ TreeStepArgs a) {
    // a warp with a game runs whole: a group past the last game replays the last one (in this warp) and stores nothing
    const int first = (blockIdx.x * blockDim.x + (threadIdx.x & ~31u)) / G;
    if (first >= a.n) return;
    const int local = (blockIdx.x * blockDim.x + threadIdx.x) / G;
    const bool own = local < a.n;
    const int g = a.g0 + (own ? local : a.n - 1);
    const int lane = LaneGroup<G>::lane();
    const int A = a.A;
    const NodePool& p = a.pool;
    if (lane == 0 && own) {
        p.range[2 * g] = INFINITY;
        p.range[2 * g + 1] = -INFINITY;
        p.ties[g] = 0;
        p.max_depth[g] = 0;
    }
    if (a.add_noise) {
        const int64_t gid = a.game_id ? a.game_id[g] : (int64_t)g;
        const int mv = a.move_index ? a.move_index[g] : 0;
        double sum = 0.0;
        if (!a.noise) {                               // drawn here: normalised Gamma(alpha) draws over the whole action space
            for (int k = lane; k < A; k += G) sum += philox_gamma(a.seed, gid, mv, k, a.noise_alpha);
            for (int off = G >> 1; off > 0; off >>= 1) sum += shfl_xor_f64(kWarp, sum, off, G);
        }
        for (int k = lane; k < A && own; k += G) {    // lane l owns the actions l, l + G, ...
            const double nz = a.noise ? a.noise[(size_t)g * A + k] : philox_gamma(a.seed, gid, mv, k, a.noise_alpha) / sum;
            if (a.trace.noise) a.trace.noise[(size_t)g * A + k] = nz;
            double* rp = p.root_prior + (size_t)g * A + k;
            *rp = __dadd_rn(__dmul_rn(*rp, __dsub_rn(1.0, a.noise_frac)), __dmul_rn(nz, a.noise_frac));
        }
    }
}

cudaError_t launch_tree_adopt_root(const TreeStepArgs& a, cudaStream_t stream) {
    int G = 4;
    while (G < a.A && G < 32) G <<= 1;
    const int grid = (a.n * G + 127) / 128;
    switch (G) {
        case 4: tree_adopt_root_kernel<4><<<grid, 128, 0, stream>>>(a); break;
        case 8: tree_adopt_root_kernel<8><<<grid, 128, 0, stream>>>(a); break;
        case 16: tree_adopt_root_kernel<16><<<grid, 128, 0, stream>>>(a); break;
        case 32: tree_adopt_root_kernel<32><<<grid, 128, 0, stream>>>(a); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_tree_step(const TreeStepArgs& a, cudaStream_t stream) {
    if (a.A > 32) return launch_tree_step_wide(a, stream);
    int G = 4;
    while (G < a.A) G <<= 1;
    const int threads = 128;
    const int games_per_cta = threads / G;
    const int grid = (a.n + games_per_cta - 1) / games_per_cta;
    // below ~4 resident warps per scheduler the kernel is latency-bound (MZ_TREE_LATENCY = 0 / 1 forces a variant: A/B switch)
    static const int forced = getenv("MZ_TREE_LATENCY") ? atoi(getenv("MZ_TREE_LATENCY")) : -1;
    const bool latency = forced >= 0 ? forced != 0 : (long)a.n * G <= 132L * 512;
    cudaError_t e = cudaSuccess;
#define MZ_TREE(GG)                                                                                 \
    case GG:                                                                                        \
        e = latency ? launch_chained(tree_step_kernel<GG, true>, dim3(grid), dim3(threads), 0, stream, a)      \
                    : launch_chained(tree_step_kernel<GG, false>, dim3(grid), dim3(threads), 0, stream, a);    \
        break;
    switch (G) {
        MZ_TREE(4) MZ_TREE(8) MZ_TREE(16) MZ_TREE(32)
        default: return cudaErrorInvalidValue;
    }
#undef MZ_TREE
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace mz
