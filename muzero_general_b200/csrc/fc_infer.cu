// Batched initial_inference / recurrent_inference for fully-connected nets (models.py:172-195),
// one lane group per sample.  Used by the step-wise search pipeline and by callers that need
// raw logits (reanalyse-style consumers, parity tests); the fused search kernel in
// fc_search.cu evaluates the same device functions in place.
#include "fc_net.cuh"
#include "kernels.h"
#include "pipeline.h"

namespace mz {

template <int G>
__global__ void __launch_bounds__(kFcThreads) fc_inference_kernel(const __grid_constant__ FcInferArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    float* s_blob = reinterpret_cast<float*>(smem);
    for (int i = threadIdx.x; i < a.net.blob_floats; i += blockDim.x) s_blob[i] = a.blob[i];
    __syncthreads();
    const int groups_per_cta = blockDim.x / G;
    const int gi = threadIdx.x / G;
    const int lane = LaneGroup<G>::lane();
    const int E = a.net.E, A = a.net.A, F = a.net.F, S = a.net.S, maxw = a.net.maxw;
    float* base = s_blob + ((a.net.blob_floats + 3) & ~3) + (size_t)gi * (4 * maxw + 4);
    float *s0 = base, *s1 = base + maxw, *s2 = base + 2 * maxw, *sh = base + 3 * maxw;   // maxw % 4 == 0

    // a warp runs while its first group has a sample (see LaneGroup); a group past the last one evaluates that one again (it
    // belongs to this warp) and stores nothing
    const int warp_first = (int)blockIdx.x * groups_per_cta + (int)(threadIdx.x & ~31u) / G;
    for (int g0 = warp_first; g0 < a.n; g0 += gridDim.x * groups_per_cta) {
        const bool own = g0 + gi - (int)(threadIdx.x & ~31u) / G < a.n;
        const int g = own ? g0 + gi - (int)(threadIdx.x & ~31u) / G : a.n - 1;
        float reward = 0.0f;
        if (a.recurrent) {
            const int act = a.action[g];
            const float* hin = a.gather_parent
                ? a.pool_hidden + ((size_t)g * a.pool_stride + a.gather_parent[g]) * E
                : a.in + (size_t)g * E;
            load_vector<G>(hin, s1, E);
            float* raw = mlp_forward<G>(a.net.dyn, s_blob, s1, s0, s1, s2, act);
            float* rl = mlp_forward<G>(a.net.rew, s_blob, raw, s0, s1, nullptr);
            if (a.reward_logits && own) for (int i = lane; i < F; i += G) a.reward_logits[(size_t)g * F + i] = rl[i];
            reward = support_to_scalar_group<G>(rl, S);
            LaneGroup<G>::sync();
            rescale_unit_range<G>(raw, sh, E);
        } else {
            load_vector<G>(a.in + (size_t)g * a.net.obs_elems, s1, a.net.obs_elems);
            float* raw = mlp_forward<G>(a.net.rep, s_blob, s1, s0, s1, s2);
            rescale_unit_range<G>(raw, sh, E);
            if (a.reward_logits && own)        // log(one-hot at the centre), models.py:176-183
                for (int i = lane; i < F; i += G) a.reward_logits[(size_t)g * F + i] = (i == S) ? 0.0f : -INFINITY;
            reward = inverse_value_transform(0.0f);
        }
        if (a.hidden && own) for (int i = lane; i < E; i += G) a.hidden[(size_t)g * E + i] = sh[i];
        if (a.pool_hidden && own)
            for (int i = lane; i < E; i += G) a.pool_hidden[((size_t)g * a.pool_stride + a.out_slot) * E + i] = sh[i];
        float* pol = mlp_forward<G>(a.net.pol, s_blob, sh, s0, s1, s2);
        if (a.policy_logits && own) for (int i = lane; i < A; i += G) a.policy_logits[(size_t)g * A + i] = pol[i];
        LaneGroup<G>::sync();
        float* vl = mlp_forward<G>(a.net.val, s_blob, sh, s0, s1, s2);
        if (a.value_logits && own) for (int i = lane; i < F; i += G) a.value_logits[(size_t)g * F + i] = vl[i];
        const float value = support_to_scalar_group<G>(vl, S);
        if (lane == 0 && own) {
            if (a.value) a.value[g] = value;
            if (a.reward) a.reward[g] = reward;
        }
        LaneGroup<G>::sync();
    }
}

// Threads of a CTA of fc_inference_kernel<G>: the most of 128, 96, 64, 32 whose groups' scratch fits next to the weight blob
// in `smem_cap` bytes of shared memory (the device's opt-in limit per block).  Host arithmetic only.
bool fc_infer_plan(int blob_floats, int maxw, int G, int n, int sm_count, size_t smem_cap, FcInferPlan* p) {
    if (G < 1 || G > 32 || 32 % G || n < 1 || sm_count < 1 || blob_floats < 0 || maxw < 1) return false;
    for (int t = kFcThreads; t >= 32; t -= 32) {
        const size_t smem = fc_infer_smem(blob_floats, maxw, t / G);
        if (smem > smem_cap) continue;
        const int groups = t / G;
        int grid = (n + groups - 1) / groups;
        if (grid > sm_count * 8) grid = sm_count * 8;
        *p = FcInferPlan{t, groups, grid, smem};
        return true;
    }
    return false;
}

template <int G>
static cudaError_t launch_infer(const FcInferArgs& a, int sm_count, size_t smem_cap, cudaStream_t stream) {
    FcInferPlan p;
    if (!fc_infer_plan(a.net.blob_floats, a.net.maxw, G, a.n, sm_count, smem_cap, &p)) return cudaErrorInvalidConfiguration;
    auto kern = fc_inference_kernel<G>;
    static size_t attr_smem = 0;
    if (attr_smem < p.smem) {
        const cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
        if (err != cudaSuccess) return err;
        attr_smem = p.smem;
    }
    kern<<<p.grid, p.threads, p.smem, stream>>>(a);
    return cudaGetLastError();
}

// The lane-group width must equal the fused search kernel's: the fp32 reductions (softmax and
// support sums) are shuffle trees over G lanes, so the same G gives bit-identical outputs.
cudaError_t launch_fc_inference(const FcInferArgs& a, int group, int sm_count, size_t smem_cap, cudaStream_t stream) {
    switch (group) {
        case 4: return launch_infer<4>(a, sm_count, smem_cap, stream);
        case 8: return launch_infer<8>(a, sm_count, smem_cap, stream);
        case 16: return launch_infer<16>(a, sm_count, smem_cap, stream);
        case 32: return launch_infer<32>(a, sm_count, smem_cap, stream);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_fc_inference_pool(const FcNet& net, const float* blob, const InferCall& c, int group, int sm_count, size_t smem_cap,
                                     cudaStream_t stream) {
    FcInferArgs a{};
    a.n = c.n; a.recurrent = c.recurrent; a.net = net; a.blob = blob; a.in = c.in; a.action = c.action;
    a.gather_parent = c.gather_parent; a.pool_hidden = c.pool_hidden; a.pool_stride = c.pool_stride; a.out_slot = c.out_slot;
    a.value_logits = c.value_logits; a.reward_logits = c.reward_logits; a.policy_logits = c.policy_logits;
    a.hidden = c.hidden; a.value = c.value; a.reward = c.reward;
    return launch_fc_inference(a, group, sm_count, smem_cap, stream);
}

}  // namespace mz
