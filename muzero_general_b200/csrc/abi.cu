// Host side of libmzb200.so: the C ABI declared in include/mzb200.h.
//
// Owns the device allocations (node pool, hidden-state pool, IO arenas, weight blobs), turns a
// reference state_dict into kernel layouts, and dispatches a batched MCTS.run to
//   - the fused persistent kernel (fc_search.cu) for fully-connected nets, or
//   - the step-wise pipeline select -> network -> expand+backup (tree_kernels.cu + the network
//     kernels) for residual nets, for teacher-forced tree tests and on MZ_FLAG_STEPWISE.
// No torch types, no exceptions across the boundary, never aborts.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <type_traits>
#include <string>
#include <vector>

#include "handle.h"
#include "cnn_stem.h"
#include "conv_wide.h"
#include "small_search.h"

using namespace mz;

static thread_local std::string g_create_error;

int mz_fail(MzHandle* h, int code, const std::string& msg) {
    if (h) h->err = msg; else g_create_error = msg;
    return code;
}

template <typename T>
static cudaError_t dev_alloc(T** p, size_t count) { return cudaMalloc(reinterpret_cast<void**>(p), count * sizeof(T) + 16); }

static void* named_buffer(MzHandle* h, const char* name, size_t bytes) {
    auto it = h->named.find(name);
    if (it != h->named.end() && it->second.second >= bytes) return it->second.first;
    if (it != h->named.end()) cudaFree(it->second.first);
    void* p = nullptr;
    if (cudaMalloc(&p, bytes + 16) != cudaSuccess) return nullptr;
    h->named[name] = {p, bytes};
    return p;
}

extern "C" int mz_abi_version(void) { return MZ_ABI_VERSION; }

extern "C" const char* mz_last_error(const MzHandle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

static int mlp_dims(const int32_t* hidden, int n_hidden, int in, int out, std::vector<int>& sizes) {
    if (n_hidden < 0 || n_hidden > MZ_MAX_LAYERS) return -1;
    sizes.clear();
    sizes.push_back(in);
    for (int i = 0; i < n_hidden; ++i) sizes.push_back(hidden[i]);
    sizes.push_back(out);
    return 0;
}

extern "C" int mz_create(const MzNetDesc* net, const MzSearchDesc* search, int device, MzHandle** out) {
    if (!net || !search || !out) return fail(nullptr, MZ_EINVAL, "mz_create: null argument");
    *out = nullptr;
    if (search->num_players > 2)       // self_play.py:429-430
        return fail(nullptr, MZ_EUNSUPPORTED, "More than two player mode not implemented.");
    if (search->num_players < 1 || search->max_games < 1 || search->num_simulations < 0)
        return fail(nullptr, MZ_EINVAL, "mz_create: bad search descriptor");
    if (net->action_space < 1 || net->action_space > MZ_MAX_ACTIONS)
        return fail(nullptr, MZ_EUNSUPPORTED, "mz_create: action_space must be in [1, 256]");
    if (net->kind != MZ_NET_FC && net->kind != MZ_NET_RESNET)
        return fail(nullptr, MZ_EUNSUPPORTED, "The network parameter should be \"fullyconnected\" or \"resnet\".");
    if (net->kind == MZ_NET_RESNET && (net->downsample < 0 || net->downsample > 2))
        return fail(nullptr, MZ_EUNSUPPORTED, "downsample should be \"resnet\" or \"CNN\".");

    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= device)
        return fail(nullptr, MZ_ECUDA, "mz_create: no such CUDA device (this library has no CPU fallback)");
    MzHandle* h = new (std::nothrow) MzHandle();
    if (!h) return fail(nullptr, MZ_ENOMEM, "mz_create: out of host memory");
    h->net = *net;
    h->search = *search;
    h->search.pb_c_table = nullptr;
    h->search.sqrt_table = nullptr;
    h->search.ucb_table = nullptr;
    h->device = device;
#define MZ_CREATE_CUDA(expr)                                                                      \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) {                                                                  \
            fail(nullptr, MZ_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));           \
            mz_destroy(h);                                                                        \
            return MZ_ECUDA;                                                                      \
        }                                                                                         \
    } while (0)
    MZ_CREATE_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    MZ_CREATE_CUDA(cudaGetDeviceProperties(&prop, device));
    h->sm_count = prop.multiProcessorCount;
    h->fc_launch.smem_per_sm = prop.sharedMemPerMultiprocessor;
    h->fc_launch.smem_reserve = prop.reservedSharedMemPerBlock;
    h->fc_launch.smem_cap = prop.sharedMemPerBlockOptin;
    MZ_CREATE_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    MZ_CREATE_CUDA(cudaEventCreate(&h->ev0));
    MZ_CREATE_CUDA(cudaEventCreate(&h->ev1));

    if (search->extra_expansions < 0) { fail(nullptr, MZ_EINVAL, "mz_create: extra_expansions < 0"); mz_destroy(h); return MZ_EINVAL; }
    // N below is the LAYOUT size of the pool and tables (room for num_simulations + 1 + extra_expansions expansions)
    const int B = search->max_games, N = search->num_simulations + search->extra_expansions, A = net->action_space;
    h->pool_n = N;
    // ---- UCB tables (self_play.py:385-390)
    std::vector<double> pbc(N + 2), sq(N + 2);
    for (int n = 0; n < N + 2; ++n) {
        pbc[n] = search->pb_c_table ? search->pb_c_table[n]
                                    : log(((double)n + search->pb_c_base + 1) / search->pb_c_base) + search->pb_c_init;
        sq[n] = search->sqrt_table ? search->sqrt_table[n] : sqrt((double)n);
    }
    MZ_CREATE_CUDA(dev_alloc(&h->d_pbc, N + 2));
    MZ_CREATE_CUDA(dev_alloc(&h->d_sqrt, N + 2));
    MZ_CREATE_CUDA(cudaMemcpy(h->d_pbc, pbc.data(), (N + 2) * 8, cudaMemcpyHostToDevice));
    MZ_CREATE_CUDA(cudaMemcpy(h->d_sqrt, sq.data(), (N + 2) * 8, cudaMemcpyHostToDevice));
    if (search->ucb_table) {
        const size_t cells = (size_t)(N + 2) * (N + 2);
        MZ_CREATE_CUDA(dev_alloc(&h->d_ucb, cells));
        MZ_CREATE_CUDA(cudaMemcpy(h->d_ucb, search->ucb_table, cells * 8, cudaMemcpyHostToDevice));
    }

    // ---- sizes
    h->obs_elems = (int64_t)net->obs_c * net->obs_h * net->obs_w;
    if (net->kind == MZ_NET_FC) {
        h->hidden_elems = net->encoding;
    } else {
        const int hh = net->downsample ? (net->obs_h + 15) / 16 : net->obs_h;
        const int hw = net->downsample ? (net->obs_w + 15) / 16 : net->obs_w;
        h->hidden_elems = (int64_t)net->channels * hh * hw;
    }
    h->pool_state_elems = h->hidden_elems;
    if (net->kind == MZ_NET_RESNET) {
        std::string e;
        h->res = resnet_create(*net, B, h->sm_count, &e);
        if (!h->res) { fail(nullptr, MZ_ECUDA, "resnet_create: " + e); mz_destroy(h); return MZ_ECUDA; }
        h->pool_state_elems = resnet_state_elems(h->res);
    }
    // ---- node pool
    const size_t slots = (size_t)B * (N + 1) * A;
    NodePool& p = h->pool;
    MZ_CREATE_CUDA(dev_alloc(&p.visit, slots));
    MZ_CREATE_CUDA(dev_alloc(&p.vsum, slots));
    MZ_CREATE_CUDA(dev_alloc(&p.mval, slots));
    MZ_CREATE_CUDA(dev_alloc(&p.reward, slots));
    MZ_CREATE_CUDA(dev_alloc(&p.prior, slots));
    MZ_CREATE_CUDA(dev_alloc(&p.expansion, slots));
    MZ_CREATE_CUDA(dev_alloc(&p.root_prior, (size_t)B * A));
    MZ_CREATE_CUDA(dev_alloc(&p.hidden, (size_t)B * (N + 1) * h->pool_state_elems));
    MZ_CREATE_CUDA(cudaMemset(p.hidden, 0, (size_t)B * (N + 1) * h->pool_state_elems * 4));   // layout padding reads as zero
    MZ_CREATE_CUDA(dev_alloc(&p.root_visit, B));
    MZ_CREATE_CUDA(dev_alloc(&p.root_vsum, B));
    MZ_CREATE_CUDA(dev_alloc(&p.root_reward, B));
    MZ_CREATE_CUDA(dev_alloc(&p.range, (size_t)B * 2));
    MZ_CREATE_CUDA(dev_alloc(&p.n_expanded, B));
    MZ_CREATE_CUDA(dev_alloc(&p.ties, B));
    MZ_CREATE_CUDA(dev_alloc(&p.max_depth, B));
    MZ_CREATE_CUDA(dev_alloc(&p.legal, (size_t)B * (MZ_MAX_ACTIONS / 32)));     // one word per game (|A| <= 32), or a stride of eight of which tree_wide.cu reads four or eight
    MZ_CREATE_CUDA(dev_alloc(&p.path, (size_t)B * (N + 2)));
    MZ_CREATE_CUDA(dev_alloc(&p.path_reward, (size_t)B * (N + 2)));
    MZ_CREATE_CUDA(dev_alloc(&p.leaf_depth, B));
    MZ_CREATE_CUDA(dev_alloc(&p.leaf_parent, B));
    MZ_CREATE_CUDA(dev_alloc(&p.leaf_action, B));
    MZ_CREATE_CUDA(dev_alloc(&p.leaf_slot, B));
    MZ_CREATE_CUDA(dev_alloc(&p.net_value, B));
    MZ_CREATE_CUDA(dev_alloc(&p.net_reward, B));
    MZ_CREATE_CUDA(dev_alloc(&p.net_policy, (size_t)B * A));
    MZ_CREATE_CUDA(cudaMemset(p.n_expanded, 0, B * sizeof(int)));

    // ---- IO arenas (sized for max_games)
    h->in_cap = (size_t)B * (h->obs_elems * 4 + A * 1 + 4 + A * 8 + 4 + 8 + 4) + 16 * 256;
    h->out_cap = (size_t)B * (A * 4 + 8 + 4 + 4 + 4 + A * 8 + 16) + 16 * 256;
    MZ_CREATE_CUDA(cudaMalloc(&h->d_in, h->in_cap));
    MZ_CREATE_CUDA(cudaMalloc(&h->d_out, h->out_cap));
    MZ_CREATE_CUDA(cudaMallocHost(&h->h_in, h->in_cap));
    MZ_CREATE_CUDA(cudaMallocHost(&h->h_out, h->out_cap));

    const char* genv = getenv("MZ_FC_GROUP");
    if (genv) h->fc_group = atoi(genv);
    else {
        int g = 8;
        while (g < A && g < 32) g <<= 1;
        if (g < 16) g = 16;
        h->fc_group = g;                     // |A| > 32: 32 lanes stride over the outputs; the search itself is step-wise
    }
    const char* tenv = getenv("MZ_FC_THREADS");
    if (tenv) h->fc_threads = atoi(tenv);
    if (h->fc_threads < 32 || h->fc_threads > kFcMaxThreads || h->fc_threads % 32) h->fc_threads = 0;
    if ((h->fc_group < A && A <= 32) || (h->fc_group != 4 && h->fc_group != 8 && h->fc_group != 16 && h->fc_group != 32)) {
        fail(nullptr, MZ_EINVAL, "mz_create: MZ_FC_GROUP must be 4, 8, 16 or 32 and >= action_space");
        mz_destroy(h);
        return MZ_EINVAL;
    }
    *out = h;
    return MZ_OK;
}

extern "C" int mz_destroy(MzHandle* h) {
    if (!h) return MZ_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    mz_selfplay_destroy(h);
    mz_reanalyse_destroy(h);
    mz_user_env_destroy(h);
    NodePool& p = h->pool;
    void* ptrs[] = {p.visit, p.vsum, p.mval, p.reward, p.prior, p.expansion, p.root_prior, p.hidden, p.root_visit, p.root_vsum,
                    p.root_reward, p.range, p.n_expanded, p.ties, p.max_depth, p.legal, p.path, p.path_reward, p.leaf_depth,
                    p.leaf_parent, p.leaf_action, p.leaf_slot, p.net_value, p.net_reward, p.net_policy, h->d_ucb, h->d_pbc, h->d_sqrt, h->d_fc_blob, h->d_in, h->d_out};
    for (void* q : ptrs) if (q) cudaFree(q);
    for (auto& kv : h->named) cudaFree(kv.second.first);
    if (h->h_in) cudaFreeHost(h->h_in);
    if (h->h_out) cudaFreeHost(h->h_out);
    mz_drop_graphs(h);
    if (h->res) resnet_destroy(h->res);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->part_fork) cudaEventDestroy(h->part_fork);
    for (int p = 0; p < MzHandle::kMaxParts; ++p) {
        if (h->part_join[p]) cudaEventDestroy(h->part_join[p]);
        if (h->part_stream[p]) cudaStreamDestroy(h->part_stream[p]);
    }
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return MZ_OK;
}

extern "C" const char* mz_numerics(const MzHandle* h) {
    if (!h) return "";
    if (h->net.kind == MZ_NET_FC) return "f32 nets + f64 tree statistics";
    return resnet_numerics(h->res);
}
extern "C" int64_t mz_hidden_elems(const MzHandle* h) { return h ? h->hidden_elems : 0; }
extern "C" int64_t mz_obs_elems(const MzHandle* h) { return h ? h->obs_elems : 0; }
extern "C" int64_t mz_launch_count(const MzHandle* h) { return h ? h->launches : 0; }
extern "C" double mz_last_search_ms(const MzHandle* h) { return h ? h->last_ms : 0.0; }
extern "C" int32_t mz_graph_partitions(const MzHandle* h) { return h ? h->graph_parts : 1; }
extern "C" int mz_fc_last_launch(const MzHandle* h, int64_t* info) {
    if (!h || !info || !h->fc_launch.launched) return 0;
    const FcLaunchInfo& l = h->fc_launch.last;
    const int64_t out[5] = {l.grid, l.block, l.group, (int64_t)l.smem, l.ctas_per_sm};
    for (int i = 0; i < 5; ++i) info[i] = out[i];
    return 1;
}

extern "C" int mz_debug_fc_prepared(const MzHandle* h, int64_t* info) {
    if (!h || !info || !h->fc_launch.prepared.valid) return 0;
    const FcPrepared& p = h->fc_launch.prepared;
    const int64_t out[7] = {p.key.n_games, p.key.group, p.key.threads, p.key.generic, p.key.one_level, p.select_levels,
                            p.fixed_shape};
    for (int i = 0; i < 7; ++i) info[i] = out[i];
    return 1;
}

// ------------------------------------------------------------------------------------------
// weights
// ------------------------------------------------------------------------------------------
static const MzTensor* find_tensor(const MzTensor* t, int n, const std::string& name) {
    for (int i = 0; i < n; ++i) if (t[i].name && name == t[i].name) return &t[i];
    return nullptr;
}

// Appends one mlp (models.py:630-642) to the blob: per Linear the weights packed [i/4][out][i%4]
// (zero padded), the bias, and - for the first dynamics layer - the one-hot rows [A][out].  t == nullptr packs zeros
// (the shapes alone, for the host-only plans).
static bool pack_mlp(const MzTensor* t, int n, const std::string& prefix, const std::vector<int>& sizes, MlpDesc& d,
                     std::vector<float>& blob, int onehot_rows, std::string* err) {
    d.n = (int)sizes.size() - 1;
    for (int l = 0; l < d.n; ++l) {
        const int in = sizes[l], out = sizes[l + 1];
        const MzTensor* w = t ? find_tensor(t, n, prefix + "." + std::to_string(2 * l) + ".weight") : nullptr;
        const MzTensor* b = t ? find_tensor(t, n, prefix + "." + std::to_string(2 * l) + ".bias") : nullptr;
        if (t && (!w || !b)) { *err = "missing tensor " + prefix + "." + std::to_string(2 * l); return false; }
        if (t && (w->numel != (int64_t)in * out || b->numel != out)) { *err = "shape mismatch for " + prefix + "." + std::to_string(2 * l); return false; }
        const int extra = (l == 0) ? onehot_rows : 0;
        const int dense = in - extra, in4 = (dense + 3) / 4;
        d.in[l] = in; d.out[l] = out; d.in_dense[l] = dense;
        while (blob.size() % 4) blob.push_back(0.0f);
        d.w_off[l] = (int)blob.size();
        blob.resize(blob.size() + (size_t)in4 * out * 4, 0.0f);
        float* dst = blob.data() + d.w_off[l];
        if (t)
            for (int o = 0; o < out; ++o)
                for (int i = 0; i < dense; ++i)
                    dst[((size_t)(i / 4) * out + o) * 4 + (i % 4)] = w->data[(size_t)o * in + i];     // torch Linear: [out][in]
        d.b_off[l] = (int)blob.size();
        if (t) blob.insert(blob.end(), b->data, b->data + out);
        else blob.resize(blob.size() + out, 0.0f);
        d.x_off[l] = -1;
        if (extra > 0) {
            d.x_off[l] = (int)blob.size();
            for (int a = 0; a < extra; ++a)
                for (int o = 0; o < out; ++o) blob.push_back(t ? w->data[(size_t)o * in + dense + a] : 0.0f);
        }
    }
    return true;
}

// The descriptors and the shared-memory blob of an FC network (nd's shape, obs_elems inputs) from torch-layout tensors, or
// of zeros when t == nullptr.
static bool fc_build_net(const MzNetDesc& nd, int obs_elems, const MzTensor* t, int n, FcNet* out, std::vector<float>* blob_out,
                  std::string* err) {
    const int E = nd.encoding, A = nd.action_space, F = 2 * nd.support_size + 1;
    if (E < 1 || A < 1 || nd.support_size < 0 || obs_elems < 1) { *err = "bad network shape"; return false; }
    FcNet fc{};
    std::vector<float>& blob = *blob_out;
    blob.clear();
    std::vector<int> sz;
    const struct { const int32_t* hidden; int n_hidden; const char* prefix; int in, out, onehot; MlpDesc* d; } mlps[] = {
        {nd.fc_representation, nd.n_fc_representation, "representation_network.module", obs_elems, E, 0, &fc.rep},
        {nd.fc_dynamics, nd.n_fc_dynamics, "dynamics_encoded_state_network.module", E + A, E, A, &fc.dyn},
        {nd.fc_reward, nd.n_fc_reward, "dynamics_reward_network.module", E, F, 0, &fc.rew},
        {nd.fc_value, nd.n_fc_value, "prediction_value_network.module", E, F, 0, &fc.val},
        {nd.fc_policy, nd.n_fc_policy, "prediction_policy_network.module", E, A, 0, &fc.pol}};
    for (const auto& m : mlps) {
        if (mlp_dims(m.hidden, m.n_hidden, m.in, m.out, sz)) { *err = "bad layers"; return false; }
        for (int w : sz) if (w < 1) { *err = "bad layers"; return false; }
        if (!pack_mlp(t, n, m.prefix, sz, *m.d, blob, m.onehot, err)) return false;
    }
    fc.blob_floats = (int)blob.size();
    fc.obs_elems = obs_elems; fc.E = E; fc.A = A; fc.S = nd.support_size; fc.F = F;
    int maxw = E > F ? E : F;
    if (A > maxw) maxw = A;
    if (obs_elems > maxw) maxw = obs_elems;
    while (blob.size() % 4) blob.push_back(0.0f);
    const MlpDesc* all[] = {&fc.rep, &fc.dyn, &fc.rew, &fc.val, &fc.pol};
    for (const MlpDesc* d : all) for (int l = 0; l < d->n; ++l) if (d->out[l] > maxw) maxw = d->out[l];
    fc.maxw = (maxw + 3) & ~3;
    *out = fc;
    return true;
}

static int load_fc_weights(MzHandle* h, const MzTensor* t, int n) {
    FcNet fc;
    std::vector<float> blob;
    std::string e;
    if (!fc_build_net(h->net, (int)h->obs_elems, t, n, &fc, &blob, &e)) return fail(h, MZ_EINVAL, "mz_load_weights: " + e);
    // every inference and every search needs the blob and at least one warp's lane groups in one CTA's shared memory
    FcInferPlan ip;
    if (!fc_infer_plan(fc.blob_floats, fc.maxw, h->fc_group, 1, h->sm_count, h->fc_launch.smem_cap, &ip))
        return fail(h, MZ_EUNSUPPORTED, "mz_load_weights: the FC network needs " +
                                            std::to_string(fc_infer_smem(fc.blob_floats, fc.maxw, 32 / h->fc_group)) +
                                            " bytes of shared memory per CTA (" + std::to_string(fc.blob_floats * 4) +
                                            " of weights and the scratch of " + std::to_string(32 / h->fc_group) +
                                            " lane groups), the device allows " + std::to_string(h->fc_launch.smem_cap));
    if (h->d_fc_blob) cudaFree(h->d_fc_blob);
    h->d_fc_blob = nullptr;
    MZ_CUDA(h, dev_alloc(&h->d_fc_blob, blob.size()));
    MZ_CUDA(h, cudaMemcpy(h->d_fc_blob, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice));
    h->fc = fc;
    h->fc_launch.prepared.valid = false;
    return MZ_OK;
}

extern "C" int mz_load_weights(MzHandle* h, const MzTensor* tensors, int32_t n) {
    if (!h || !tensors || n <= 0) return fail(h, MZ_EINVAL, "mz_load_weights: null argument");
    MZ_CUDA(h, cudaSetDevice(h->device));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    mz_drop_graphs(h);                 // weight buffers move
    int rc;
    if (h->net.kind == MZ_NET_FC) {
        rc = load_fc_weights(h, tensors, n);
    } else {
        std::string e;
        rc = resnet_load_weights(h->res, tensors, n, &e);
        if (rc) return fail(h, rc, "mz_load_weights: " + e);
    }
    if (rc == MZ_OK) h->weights_loaded = true;
    return rc;
}

// ------------------------------------------------------------------------------------------
// search
// ------------------------------------------------------------------------------------------
struct Arena {
    size_t off = 0;
    size_t take(size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; }
};

template <typename T>
static const T* stage_in(MzHandle* h, Arena& ar, const T* src, size_t count) {
    if (!src) return nullptr;
    const size_t o = ar.take(count * sizeof(T));
    memcpy(h->h_in + o, src, count * sizeof(T));
    return reinterpret_cast<const T*>(h->d_in + o);
}

struct OutSlot { void* user; size_t off, bytes; };
template <typename T>
static T* stage_out(MzHandle* h, Arena& ar, T* user, size_t count, std::vector<OutSlot>& slots) {
    if (!user) return nullptr;
    const size_t o = ar.take(count * sizeof(T));
    slots.push_back({user, o, count * sizeof(T)});
    return reinterpret_cast<T*>(h->d_out + o);
}

template <typename T>
static int debug_in(MzHandle* h, const char* name, const T* src, size_t count, int mem, const T** out) {
    *out = nullptr;
    if (!src) return MZ_OK;
    if (mem == MZ_MEM_DEVICE) { *out = src; return MZ_OK; }
    void* d = named_buffer(h, name, count * sizeof(T));
    if (!d) return fail(h, MZ_ENOMEM, std::string("out of device memory for ") + name);
    MZ_CUDA(h, cudaMemcpyAsync(d, src, count * sizeof(T), cudaMemcpyHostToDevice, h->stream));
    *out = reinterpret_cast<const T*>(d);
    return MZ_OK;
}

struct DebugOut { void* user; void* dev; size_t bytes; };
template <typename T>
static int debug_out(MzHandle* h, const char* name, T* user, size_t count, int mem, T** out, std::vector<DebugOut>& outs) {
    *out = nullptr;
    if (!user) return MZ_OK;
    if (mem == MZ_MEM_DEVICE) { *out = user; return MZ_OK; }
    void* d = named_buffer(h, name, count * sizeof(T));
    if (!d) return fail(h, MZ_ENOMEM, std::string("out of device memory for ") + name);
    outs.push_back({user, d, count * sizeof(T)});
    *out = reinterpret_cast<T*>(d);
    return MZ_OK;
}

// The x3 towers' range guard fired: fp32 CUDA-core towers from now on (the hidden-state pool is large enough for the
// dense layout; a captured graph refers to the old kernels and is dropped).
void mz_switch_to_strict(MzHandle* h) {
    if (!h->res) return;
    resnet_use_strict(h->res);
    h->pool_state_elems = resnet_state_elems(h->res);
    mz_drop_graphs(h);
    h->range_fallbacks += 1;
}

void mz_drop_graphs(MzHandle* h) {
    for (auto& e : h->graphs) if (e.exec) cudaGraphExecDestroy(e.exec);
    h->graphs.clear();
}

// Number of parallel branches the captured graph of a search over n games is split into (1 = no split).
// MZ_PARTS = 1 switches the partitioned replay off, 2..4 forces that many branches wherever the kernels allow it.
static int search_partitions(MzHandle* h, int n, int continue_from) {
    const char* penv = getenv("MZ_PARTS");
    const int forced = penv ? atoi(penv) : 0;
    if (forced == 1 || continue_from > 0 || h->net.kind != MZ_NET_RESNET || h->net.action_space > 32 || !h->res) return 1;
    if (!resnet_can_partition(h->res)) return 1;
    // default: two branches, four from 1024 games on
    int parts = forced > 1 ? std::min(forced, (int)MzHandle::kMaxParts) : (n >= 1024 ? 4 : 2);
    if (forced <= 1 && !resnet_uses_tensor_cores(h->res)) return 1;          // default: the tensor-core towers only
    while (parts > 1 && n < parts * 64) --parts;
    if (parts < 2) return 1;
    for (int p = 1; p < parts; ++p) {
        if (!h->part_stream[p] && cudaStreamCreateWithFlags(&h->part_stream[p], cudaStreamNonBlocking) != cudaSuccess) return 1;
        if (!h->part_join[p] && cudaEventCreateWithFlags(&h->part_join[p], cudaEventDisableTiming) != cudaSuccess) return 1;
    }
    if (!h->part_fork && cudaEventCreateWithFlags(&h->part_fork, cudaEventDisableTiming) != cudaSuccess) return 1;
    return parts;
}

// ------------------------------------------------------------------------------------------
// One batched search on device buffers (no synchronisation): fused FC kernel or step-wise pipeline.
// ------------------------------------------------------------------------------------------
int mz_dispatch_search(MzHandle* h, const SearchCall& call, bool teacher, bool trace, int flags) {
    const int n = call.n, N = h->search.num_simulations, A = h->net.action_space;
    int rc;
    if (h->search.extra_expansions > 0 || A > 32) flags |= MZ_FLAG_STEPWISE;     // the fused FC kernel: N + 1 expansions, one lane per action
    SearchCall cont = call;
    cont.continue_from = (flags & MZ_FLAG_CONTINUE) ? h->imported_expansions : 0;
    const SearchCall& call_ = cont;
    const bool fused = (h->net.kind == MZ_NET_FC || teacher) && !(flags & MZ_FLAG_STEPWISE);
    if (fused) {
        FcSearchArgs a{};
        a.n_games = n; a.N = N; a.A = A; a.P = h->search.num_players; a.threads = h->fc_threads;
        a.discount = h->search.discount; a.noise_frac = h->search.root_exploration_fraction; a.noise_alpha = h->search.root_dirichlet_alpha; a.seed = h->search.seed;
        a.pbc = h->d_pbc; a.sqrtn = h->d_sqrt; a.ucb = h->d_ucb;
        a.net = h->fc; a.blob = h->d_fc_blob;
        if (teacher) { a.net.E = 1; a.net.maxw = 4; a.net.blob_floats = 0; a.net.A = A; }
        a.obs = call.obs; a.legal_mask = call.legal_mask; a.to_play = call.to_play; a.add_noise = call.add_noise;
        a.noise = call.noise; a.first_index = call.first_index; a.game_id = call.game_id; a.move_index = call.move_index;
        a.visit_counts = call.visit_counts; a.root_value = call.root_value; a.root_predicted_value = call.root_predicted_value;
        a.max_tree_depth = call.max_tree_depth; a.tie_count = call.tie_count; a.root_priors = call.root_priors;
        a.value_range = call.value_range; a.teacher = call.teacher; a.trace = call.trace;
        if (call.keep_tree) a.pool = h->pool;
        cudaError_t e = launch_fc_search(a, h->fc_group, teacher, h->sm_count, &h->fc_launch, h->stream);
        if (e == cudaErrorInvalidConfiguration) {
            // the tree does not fit in shared memory next to the weights: use the HBM node pool
            (void)cudaGetLastError();
            rc = run_stepwise_search(h->net, h->search, h->pool_n, h->pool, h->d_pbc, h->d_sqrt, h->d_ucb, h->fc, h->d_fc_blob, h->res, call_,
                                     h->fc_group, h->sm_count, h->fc_launch.smem_cap, h->stream, &h->launches, &h->err);
            if (rc) return rc;
        } else if (e != cudaSuccess) {
            return fail(h, MZ_ECUDA, std::string("fc_search launch: ") + cudaGetErrorString(e));
        } else {
            h->launches += 1;
        }
    } else {
        // The step-wise pipeline is 16 small launches per simulation: replay it as a CUDA graph once the
        // same argument set has been seen twice (first call runs eagerly so lazy attribute setup and
        // allocations happen outside capture).  Debug modes (teacher / trace) always run eagerly.
        const bool graphable = !teacher && !trace && !kt_enabled() && getenv("MZ_NO_GRAPH") == nullptr;
        // Result pointers must not be part of a graph's identity: a caller that allocates its result arrays per call (the
        // Python engine with device memory does) would never hit the cache.  The pipeline writes into the handle's own
        // output arena and a few small device-to-device copies behind the graph hand the results over.
        struct ResultCopy { void* dst; const void* src; size_t bytes; };
        ResultCopy copies[8];
        int n_copies = 0;
        if (graphable) {
            Arena ar;
            const unsigned char* lo = h->d_out;
            const unsigned char* hi = h->d_out + h->out_cap;
            auto redirect = [&](auto*& ptr, size_t count) {
                using T = std::remove_reference_t<decltype(*ptr)>;
                const unsigned char* p8 = reinterpret_cast<const unsigned char*>(ptr);
                if (!ptr || (p8 >= lo && p8 < hi)) return;               // absent, or already in the arena (host-memory calls)
                const size_t o = ar.take(count * sizeof(T));
                if (ar.off > h->out_cap) { ar.off = o; return; }         // (cannot happen: the arena is sized for max_games)
                copies[n_copies++] = {ptr, h->d_out + o, count * sizeof(T)};
                ptr = reinterpret_cast<T*>(h->d_out + o);
            };
            redirect(cont.visit_counts, (size_t)n * A);
            redirect(cont.root_value, (size_t)n);
            redirect(cont.root_predicted_value, (size_t)n);
            redirect(cont.max_tree_depth, (size_t)n);
            redirect(cont.tie_count, (size_t)n);
            redirect(cont.root_priors, (size_t)n * A);
            redirect(cont.value_range, (size_t)n * 2);
        }
        uint64_t key = 1469598103934665603ull;
        auto mix = [&](uint64_t v) { key = (key ^ v) * 1099511628211ull; };
        const void* ptrs[] = {call_.obs, call_.legal_mask, call_.to_play, call_.noise, call_.first_index, call_.game_id,
                              call_.move_index, call_.visit_counts, call_.root_value, call_.root_predicted_value,
                              call_.max_tree_depth, call_.tie_count, call_.root_priors, call_.value_range};
        for (const void* q : ptrs) mix((uint64_t)(uintptr_t)q);
        mix((uint64_t)n); mix((uint64_t)call.add_noise); mix((uint64_t)call.keep_tree); mix((uint64_t)call_.continue_from);
        auto run = [&](const SearchCall& sc, cudaStream_t st) {
            return run_stepwise_search(h->net, h->search, h->pool_n, h->pool, h->d_pbc, h->d_sqrt, h->d_ucb, h->fc, h->d_fc_blob, h->res, sc,
                                       h->fc_group, h->sm_count, h->fc_launch.smem_cap, st, &h->launches, &h->err);
        };
        auto eager = [&]() { return run(call_, h->stream); };
        // Partitioned replay.  A simulation is a chain of dependent kernels (tower -> heads -> tower -> heads -> tree step) and
        // the tensor-core towers leave the SMs they do not fill - and every SM during the heads / tree kernels - idle.  Games
        // are independent, so the captured graph runs the simulations of P disjoint game ranges as P parallel branches: the
        // towers of one range overlap the heads and tree steps of the others.  Every array stays addressed by the global
        // game index, so the arithmetic per game - and every result - is exactly that of the whole-batch call.
        const int parts = search_partitions(h, n, call_.continue_from);
        auto partitioned = [&]() -> int {
            SearchCall root = call_;
            root.phases = kPhaseRoot;
            int rc2 = run(root, h->stream);
            if (rc2) return rc2;
            if (cudaEventRecord(h->part_fork, h->stream) != cudaSuccess) return fail(h, MZ_ECUDA, "partitioned replay: fork");
            const int per = partition_games(n, parts);
            for (int p = 0; p < parts; ++p) {
                SearchCall sc = call_;
                sc.phases = kPhaseSims;
                sc.g0 = p * per;
                sc.n = std::min(per, n - sc.g0);
                if (sc.n <= 0) continue;
                cudaStream_t st = p == 0 ? h->stream : h->part_stream[p];
                if (p > 0 && cudaStreamWaitEvent(st, h->part_fork, 0) != cudaSuccess) return fail(h, MZ_ECUDA, "partitioned replay: fork wait");
                if ((rc2 = run(sc, st))) return rc2;
                if (p > 0) {
                    if (cudaEventRecord(h->part_join[p], st) != cudaSuccess || cudaStreamWaitEvent(h->stream, h->part_join[p], 0) != cudaSuccess)
                        return fail(h, MZ_ECUDA, "partitioned replay: join");
                }
            }
            return MZ_OK;
        };
        MzHandle::SearchGraph* gr = nullptr;
        if (graphable) {
            h->graph_tick += 1;
            for (auto& e : h->graphs) if (e.key == key) gr = &e;
            if (!gr) {
                if ((int)h->graphs.size() < MzHandle::kMaxGraphs) {
                    h->graphs.emplace_back();
                    gr = &h->graphs.back();
                } else {
                    gr = &h->graphs[0];
                    for (auto& e : h->graphs) if (e.used < gr->used) gr = &e;
                    if (gr->exec) cudaGraphExecDestroy(gr->exec);
                    *gr = MzHandle::SearchGraph{};
                }
                gr->key = key;
            }
            gr->used = h->graph_tick;
        }
        if (gr && gr->exec) {
            MZ_CUDA(h, cudaGraphLaunch(gr->exec, h->stream));
            h->launches += gr->launches;
            h->graph_parts = gr->parts;
        } else if (gr && gr->seen >= 1) {
            const int64_t l0 = h->launches;
            MZ_CUDA(h, cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
            rc = parts > 1 ? partitioned() : eager();
            cudaGraph_t graph = nullptr;
            cudaError_t ce = cudaStreamEndCapture(h->stream, &graph);
            if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
            if (ce != cudaSuccess) return fail(h, MZ_ECUDA, std::string("graph capture: ") + cudaGetErrorString(ce));
            ce = cudaGraphInstantiate(&gr->exec, graph, 0);
            cudaGraphDestroy(graph);
            if (ce != cudaSuccess) { gr->exec = nullptr; return fail(h, MZ_ECUDA, std::string("graph instantiate: ") + cudaGetErrorString(ce)); }
            gr->launches = h->launches - l0;
            gr->parts = parts;
            h->graph_parts = parts;
            MZ_CUDA(h, cudaGraphLaunch(gr->exec, h->stream));
        } else {
            rc = eager();
            if (rc) return rc;
            if (gr) gr->seen += 1;
            h->graph_parts = 1;
        }
        for (int i = 0; i < n_copies; ++i)
            MZ_CUDA(h, cudaMemcpyAsync(copies[i].dst, copies[i].src, copies[i].bytes, cudaMemcpyDeviceToDevice, h->stream));
    }
    return MZ_OK;
}

// The handle's device current on the calling thread (cudaSetDevice only when another one is).
static int use_device(MzHandle* h) {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != h->device) MZ_CUDA(h, cudaSetDevice(h->device));
    return MZ_OK;
}

// Enqueues the search between the handle's two events, then the D2H copies of a host-memory call (out_bytes of the
// output arena, the debug outputs).
static int enqueue_search(MzHandle* h, const SearchCall& call, bool teacher, bool trace, int flags, size_t out_bytes,
                          const std::vector<DebugOut>& dbg_outs) {
    int rc;
    // each debug output is copied back whole, and the search leaves some entries unwritten (trace actions past a leaf's
    // depth): those read 0, not whatever the device buffer held before (an earlier search, another allocation)
    for (const DebugOut& d : dbg_outs) MZ_CUDA(h, cudaMemsetAsync(d.dev, 0, d.bytes, h->stream));
    MZ_CUDA(h, cudaEventRecord(h->ev0, h->stream));
    if ((rc = mz_dispatch_search(h, call, teacher, trace, flags))) return rc;
    h->host_ns[1] = mz_host_ns();
    MZ_CUDA(h, cudaEventRecord(h->ev1, h->stream));
    if (out_bytes) MZ_CUDA(h, cudaMemcpyAsync(h->h_out, h->d_out, out_bytes, cudaMemcpyDeviceToHost, h->stream));
    for (const DebugOut& d : dbg_outs)
        MZ_CUDA(h, cudaMemcpyAsync(d.user, d.dev, d.bytes, cudaMemcpyDeviceToHost, h->stream));
    return MZ_OK;
}

// Waits for the search enqueue_search enqueued with the same arguments; a search whose tensor-core towers left the fp16
// range is redone on the fp32 towers.  Sets last_ms.
static int wait_search(MzHandle* h, const SearchCall& call, bool teacher, bool trace, int flags, size_t out_bytes,
                       const std::vector<DebugOut>& dbg_outs) {
    int rc;
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    h->host_ns[2] = mz_host_ns();
    if (h->res && !teacher && resnet_take_saturations(h->res, h->stream) > 0) {
        // an activation left the fp16 range inside the tensor-core towers: the results above are outside the accuracy
        // contract.  Switch this handle to the fp32 CUDA-core towers for good and redo the search.
        mz_switch_to_strict(h);
        if ((rc = enqueue_search(h, call, teacher, trace, flags, out_bytes, dbg_outs))) return rc;
        MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, h->ev0, h->ev1) == cudaSuccess) h->last_ms = ms;
    return MZ_OK;
}

extern "C" int mz_search(MzHandle* h, const MzSearchIO* io) {
    if (!h || !io) return fail(h, MZ_EINVAL, "mz_search: null argument");
    h->host_ns[0] = mz_host_ns();
    const int n = io->n_games, N = h->search.num_simulations, A = h->net.action_space;
    if (n < 1 || n > h->search.max_games) return fail(h, MZ_EINVAL, "mz_search: n_games out of range");
    const bool teacher = io->teacher != nullptr;
    if (!teacher && !h->weights_loaded) return fail(h, MZ_ESTATE, "mz_search: weights not loaded");
    const bool cont = (io->flags & MZ_FLAG_CONTINUE) != 0;
    if (!teacher && !io->obs && !cont) return fail(h, MZ_EINVAL, "mz_search: obs is null");
    if (cont) {
        if (n != 1) return fail(h, MZ_EINVAL, "mz_search: MZ_FLAG_CONTINUE takes one game");
        if (h->imported_expansions < 1) return fail(h, MZ_ESTATE, "mz_search: MZ_FLAG_CONTINUE without mz_import_tree");
        if (h->imported_expansions + h->search.num_simulations > h->pool_n + 1)
            return fail(h, MZ_EINVAL, "mz_search: the imported tree plus num_simulations exceeds the pool (raise extra_expansions)");
    }
    int rc;
    if ((rc = use_device(h))) return rc;

    SearchCall call{};
    call.n = n;
    std::vector<OutSlot> outs;
    std::vector<DebugOut> dbg_outs;
    const bool host = io->mem == MZ_MEM_HOST;
    if (host) {
        Arena ai, ao;
        call.obs = (teacher || cont) ? nullptr : stage_in(h, ai, io->obs, (size_t)n * h->obs_elems);
        call.legal_mask = stage_in(h, ai, io->legal_mask, (size_t)n * A);
        call.to_play = stage_in(h, ai, io->to_play, n);
        call.noise = stage_in(h, ai, io->add_exploration_noise ? io->noise : nullptr, (size_t)n * A);
        call.first_index = stage_in(h, ai, io->first_index, n);
        call.game_id = stage_in(h, ai, io->game_id, n);
        call.move_index = stage_in(h, ai, io->move_index, n);
        if (ai.off > h->in_cap) return fail(h, MZ_EINVAL, "mz_search: input arena overflow");
        if (ai.off) MZ_CUDA(h, cudaMemcpyAsync(h->d_in, h->h_in, ai.off, cudaMemcpyHostToDevice, h->stream));
        call.visit_counts = stage_out(h, ao, io->visit_counts, (size_t)n * A, outs);
        call.root_value = stage_out(h, ao, io->root_value, n, outs);
        call.root_predicted_value = stage_out(h, ao, io->root_predicted_value, n, outs);
        call.max_tree_depth = stage_out(h, ao, io->max_tree_depth, n, outs);
        call.tie_count = stage_out(h, ao, io->tie_count, n, outs);
        call.root_priors = stage_out(h, ao, io->root_priors, (size_t)n * A, outs);
        call.value_range = stage_out(h, ao, io->value_range, (size_t)n * 2, outs);
        if (ao.off > h->out_cap) return fail(h, MZ_EINVAL, "mz_search: output arena overflow");
        call.out_bytes = ao.off;
    } else {
        call.obs = io->obs; call.legal_mask = io->legal_mask; call.to_play = io->to_play;
        call.noise = io->add_exploration_noise ? io->noise : nullptr;
        call.first_index = io->first_index; call.game_id = io->game_id; call.move_index = io->move_index;
        call.visit_counts = io->visit_counts; call.root_value = io->root_value;
        call.root_predicted_value = io->root_predicted_value; call.max_tree_depth = io->max_tree_depth;
        call.tie_count = io->tie_count; call.root_priors = io->root_priors; call.value_range = io->value_range;
    }
    call.add_noise = io->add_exploration_noise;
    if (teacher) {
        const MzTeacher& t = *io->teacher;
        if ((rc = debug_in(h, "t.root_value", t.root_value, n, io->mem, &call.teacher.root_value))) return rc;
        if ((rc = debug_in(h, "t.root_reward", t.root_reward, n, io->mem, &call.teacher.root_reward))) return rc;
        if ((rc = debug_in(h, "t.root_priors", t.root_priors, (size_t)n * A, io->mem, &call.teacher.root_priors))) return rc;
        if ((rc = debug_in(h, "t.value", t.value, (size_t)n * N, io->mem, &call.teacher.value))) return rc;
        if ((rc = debug_in(h, "t.reward", t.reward, (size_t)n * N, io->mem, &call.teacher.reward))) return rc;
        if ((rc = debug_in(h, "t.priors", t.priors, (size_t)n * N * A, io->mem, &call.teacher.priors))) return rc;
        if (!call.teacher.root_value || !call.teacher.root_reward || !call.teacher.root_priors ||
            (N > 0 && (!call.teacher.value || !call.teacher.reward || !call.teacher.priors)))
            return fail(h, MZ_EINVAL, "mz_search: incomplete teacher table");
    }
    if (io->trace) {
        // the kernels address a game's trace rows by the pool's layout size, the caller's arrays hold num_simulations rows
        // per game: the two agree for one game, and for any number when the pool has no extra room
        if (n > 1 && h->search.extra_expansions > 0)
            return fail(h, MZ_EINVAL, "mz_search: a trace of more than one game needs a handle with extra_expansions = 0");
        const MzTrace& t = *io->trace;
        const int D = t.max_depth;
        call.trace.max_depth = D;
        if ((rc = debug_out(h, "r.depth", t.depth, (size_t)n * N, io->mem, &call.trace.depth, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.actions", t.actions, (size_t)n * N * D, io->mem, &call.trace.actions, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.value", t.value, (size_t)n * N, io->mem, &call.trace.value, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.reward", t.reward, (size_t)n * N, io->mem, &call.trace.reward, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.priors", t.priors, (size_t)n * N * A, io->mem, &call.trace.priors, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.root_priors_raw", t.root_priors_raw, (size_t)n * A, io->mem, &call.trace.root_priors_raw, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.root_reward", t.root_reward, n, io->mem, &call.trace.root_reward, dbg_outs))) return rc;
        if ((rc = debug_out(h, "r.noise", t.noise, (size_t)n * A, io->mem, &call.trace.noise, dbg_outs))) return rc;
        if (call.trace.depth && (!call.trace.actions || !call.trace.value || !call.trace.reward || !call.trace.priors))
            return fail(h, MZ_EINVAL, "mz_search: trace needs depth, actions, value, reward and priors together");
    }
    call.keep_tree = (io->flags & MZ_FLAG_KEEP_TREE) != 0;

    const bool trace = io->trace != nullptr;
    const size_t out_bytes = host ? call.out_bytes : 0;
    if ((rc = enqueue_search(h, call, teacher, trace, io->flags, out_bytes, dbg_outs))) return rc;
    if ((rc = wait_search(h, call, teacher, trace, io->flags, out_bytes, dbg_outs))) return rc;
    for (const OutSlot& s : outs) memcpy(s.user, h->h_out + s.off, s.bytes);
    h->host_ns[3] = mz_host_ns();
    return MZ_OK;
}

// The lean entry point of a search on device memory, in two calls so that the caller's own work overlaps the search:
// mz_search_device enqueues (no staging, no debug outputs; the fused FC route goes straight to the launch its prepared
// state holds, launch_fc_search), mz_search_device_wait waits.  Every route is mz_search's.
extern "C" int mz_search_device(MzHandle* h, MzDeviceSearchIO* io) {
    if (!h || !io) return fail(h, MZ_EINVAL, "mz_search_device: null argument");
    h->host_ns[0] = mz_host_ns();
    const int n = io->n_games;
    if (h->device_pending) return fail(h, MZ_ESTATE, "mz_search_device: the previous search was not waited for");
    if (n < 1 || n > h->search.max_games) return fail(h, MZ_EINVAL, "mz_search_device: n_games out of range");
    if (!h->weights_loaded) return fail(h, MZ_ESTATE, "mz_search_device: weights not loaded");
    if (!io->obs) return fail(h, MZ_EINVAL, "mz_search_device: obs is null");
    int rc;
    if ((rc = use_device(h))) return rc;
    SearchCall& call = h->device_call;
    call = SearchCall{};
    call.n = n;
    call.obs = io->obs; call.legal_mask = io->legal_mask; call.to_play = io->to_play;
    call.add_noise = io->add_exploration_noise;
    call.noise = io->add_exploration_noise ? io->noise : nullptr;
    call.first_index = io->first_index; call.game_id = io->game_id; call.move_index = io->move_index;
    call.visit_counts = io->visit_counts; call.root_value = io->root_value;
    call.root_predicted_value = io->root_predicted_value; call.max_tree_depth = io->max_tree_depth;
    call.tie_count = io->tie_count; call.root_priors = io->root_priors; call.value_range = io->value_range;
    if ((rc = enqueue_search(h, call, false, false, 0, 0, {}))) return rc;
    h->device_pending = true;
    return MZ_OK;
}

extern "C" int mz_search_device_wait(MzHandle* h, MzDeviceSearchIO* io) {
    if (!h || !io) return fail(h, MZ_EINVAL, "mz_search_device_wait: null argument");
    if (!h->device_pending) return fail(h, MZ_ESTATE, "mz_search_device_wait: no search enqueued by mz_search_device");
    h->device_pending = false;
    int rc;
    if ((rc = use_device(h))) return rc;
    if ((rc = wait_search(h, h->device_call, false, false, 0, 0, {}))) return rc;
    io->device_ms = h->last_ms;
    h->host_ns[3] = mz_host_ns();
    return MZ_OK;
}

extern "C" int mz_debug_host_split(const MzHandle* h, int64_t* out) {
    if (!h || !out) return MZ_EINVAL;
    for (int i = 0; i < 4; ++i) out[i] = h->host_ns[i];
    return MZ_OK;
}

// ------------------------------------------------------------------------------------------
// network entry points
// ------------------------------------------------------------------------------------------
int mz_network_enqueue(MzHandle* h, const InferCall& c) {
    if (h->net.kind == MZ_NET_FC) {
        FcInferArgs a{};
        a.n = c.n; a.recurrent = c.recurrent; a.net = h->fc; a.blob = h->d_fc_blob; a.in = c.in; a.action = c.action;
        a.value_logits = c.value_logits; a.reward_logits = c.reward_logits; a.policy_logits = c.policy_logits;
        a.hidden = c.hidden; a.value = c.value; a.reward = c.reward;
        cudaError_t e = launch_fc_inference(a, h->fc_group, h->sm_count, h->fc_launch.smem_cap, h->stream);
        if (e != cudaSuccess) return fail(h, MZ_ECUDA, std::string("fc_inference launch: ") + cudaGetErrorString(e));
        h->launches += 1;
        return MZ_OK;
    }
    std::string e;
    const int rc = resnet_inference(h->res, c, h->stream, &h->launches, &e);
    return rc ? fail(h, rc, "resnet_inference: " + e) : MZ_OK;
}

int mz_network_guard(MzHandle* h, const InferCall& c) {
    if (!h->res || resnet_take_saturations(h->res, h->stream) == 0) return MZ_OK;
    mz_switch_to_strict(h);
    return mz_network_enqueue(h, c);
}

static int run_inference(MzHandle* h, int n, int mem, const float* in, const int32_t* action, const MzInferenceOut* out,
                         bool recurrent) {
    if (!h || !in || !out) return fail(h, MZ_EINVAL, "inference: null argument");
    if (!h->weights_loaded) return fail(h, MZ_ESTATE, "inference: weights not loaded");
    if (n < 1) return fail(h, MZ_EINVAL, "inference: n < 1");
    if (recurrent && !action) return fail(h, MZ_EINVAL, "recurrent_inference: action is null");
    MZ_CUDA(h, cudaSetDevice(h->device));
    const int A = h->net.action_space, F = 2 * h->net.support_size + 1;
    const size_t in_elems = recurrent ? (size_t)h->hidden_elems : (size_t)h->obs_elems;
    std::vector<DebugOut> outs;
    InferCall c{};
    c.n = n; c.recurrent = recurrent;
    int rc;
    if ((rc = debug_in(h, "i.in", in, (size_t)n * in_elems, mem, &c.in))) return rc;
    if ((rc = debug_in(h, "i.action", action, n, mem, &c.action))) return rc;
    if ((rc = debug_out(h, "i.vl", out->value_logits, (size_t)n * F, mem, &c.value_logits, outs))) return rc;
    if ((rc = debug_out(h, "i.rl", out->reward_logits, (size_t)n * F, mem, &c.reward_logits, outs))) return rc;
    if ((rc = debug_out(h, "i.pl", out->policy_logits, (size_t)n * A, mem, &c.policy_logits, outs))) return rc;
    if ((rc = debug_out(h, "i.h", out->hidden, (size_t)n * h->hidden_elems, mem, &c.hidden, outs))) return rc;
    if ((rc = debug_out(h, "i.v", out->value, n, mem, &c.value, outs))) return rc;
    if ((rc = debug_out(h, "i.r", out->reward, n, mem, &c.reward, outs))) return rc;
    if ((rc = mz_network_enqueue(h, c))) return rc;
    if ((rc = mz_network_guard(h, c))) return rc;
    for (const DebugOut& d : outs)
        MZ_CUDA(h, cudaMemcpyAsync(d.user, d.dev, d.bytes, cudaMemcpyDeviceToHost, h->stream));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    return MZ_OK;
}

extern "C" int mz_initial_inference(MzHandle* h, int32_t n, int32_t mem, const float* obs, const MzInferenceOut* out) {
    return run_inference(h, n, mem, obs, nullptr, out, false);
}

extern "C" int mz_recurrent_inference(MzHandle* h, int32_t n, int32_t mem, const float* hidden, const int32_t* action,
                                      const MzInferenceOut* out) {
    return run_inference(h, n, mem, hidden, action, out, true);
}

// ------------------------------------------------------------------------------------------
// tree export
// ------------------------------------------------------------------------------------------
extern "C" int mz_export_tree(MzHandle* h, int32_t game, MzTreeExport* out) {
    if (!h || !out) return fail(h, MZ_EINVAL, "mz_export_tree: null argument");
    if (game < 0 || game >= h->search.max_games) return fail(h, MZ_EINVAL, "mz_export_tree: game out of range");
    MZ_CUDA(h, cudaSetDevice(h->device));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    const int N = h->pool_n, A = h->net.action_space;
    const size_t S = (size_t)(N + 1) * A, base = (size_t)game * S;
    const NodePool& p = h->pool;
    int nexp = 0;
    MZ_CUDA(h, cudaMemcpy(&nexp, p.n_expanded + game, 4, cudaMemcpyDeviceToHost));
    if (nexp < 1) return fail(h, MZ_ESTATE, "mz_export_tree: no tree kept for this game (use MZ_FLAG_KEEP_TREE)");
    out->n_expansions = nexp;
    const size_t used = (size_t)nexp * A;
    if (out->child_visit) MZ_CUDA(h, cudaMemcpy(out->child_visit, p.visit + base, used * 4, cudaMemcpyDeviceToHost));
    if (out->child_value_sum) MZ_CUDA(h, cudaMemcpy(out->child_value_sum, p.vsum + base, used * 8, cudaMemcpyDeviceToHost));
    if (out->child_reward) MZ_CUDA(h, cudaMemcpy(out->child_reward, p.reward + base, used * 4, cudaMemcpyDeviceToHost));
    if (out->child_expansion) MZ_CUDA(h, cudaMemcpy(out->child_expansion, p.expansion + base, used * 4, cudaMemcpyDeviceToHost));
    if (out->child_prior) {
        std::vector<float> pf(used);
        std::vector<double> rp(A);
        MZ_CUDA(h, cudaMemcpy(pf.data(), p.prior + base, used * 4, cudaMemcpyDeviceToHost));
        MZ_CUDA(h, cudaMemcpy(rp.data(), p.root_prior + (size_t)game * A, A * 8, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < used; ++i) out->child_prior[i] = (i < (size_t)A) ? rp[i] : (double)pf[i];
    }
    if (out->hidden) {
        const float* src = p.hidden + (size_t)game * (N + 1) * h->pool_state_elems;
        if (h->net.kind == MZ_NET_RESNET) {
            void* tmp = named_buffer(h, "x.hidden", (size_t)nexp * h->hidden_elems * 4);
            if (!tmp) return fail(h, MZ_ENOMEM, "mz_export_tree: out of device memory");
            if (resnet_states_to_nchw(h->res, src, nexp, (float*)tmp, h->stream)) return fail(h, MZ_ECUDA, "mz_export_tree: layout conversion failed");
            MZ_CUDA(h, cudaStreamSynchronize(h->stream));
            src = (const float*)tmp;
        }
        MZ_CUDA(h, cudaMemcpy(out->hidden, src, (size_t)nexp * h->hidden_elems * 4, cudaMemcpyDeviceToHost));
    }
    MZ_CUDA(h, cudaMemcpy(&out->root_visit, p.root_visit + game, 4, cudaMemcpyDeviceToHost));
    MZ_CUDA(h, cudaMemcpy(&out->root_value_sum, p.root_vsum + game, 8, cudaMemcpyDeviceToHost));
    MZ_CUDA(h, cudaMemcpy(&out->root_reward, p.root_reward + game, 4, cudaMemcpyDeviceToHost));
    return MZ_OK;
}

// ------------------------------------------------------------------------------------------
// tree import (override_root_with, self_play.py:275-277)
// ------------------------------------------------------------------------------------------
extern "C" int mz_import_tree(MzHandle* h, int32_t game, const MzTreeExport* t) {
    if (!h || !t) return fail(h, MZ_EINVAL, "mz_import_tree: null argument");
    if (game < 0 || game >= h->search.max_games) return fail(h, MZ_EINVAL, "mz_import_tree: game out of range");
    const int N = h->pool_n, A = h->net.action_space, K = t->n_expansions;
    if (K < 1 || K > N + 1) return fail(h, MZ_EINVAL, "mz_import_tree: n_expansions does not fit the pool (raise extra_expansions)");
    if (!t->child_visit || !t->child_value_sum || !t->child_reward || !t->child_prior || !t->child_expansion)
        return fail(h, MZ_EINVAL, "mz_import_tree: incomplete tree");
    MZ_CUDA(h, cudaSetDevice(h->device));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    const size_t S = (size_t)(N + 1) * A, base = (size_t)game * S, used = (size_t)K * A;
    const NodePool& p = h->pool;
    std::vector<float> prior(used);
    std::vector<double> mval(used, 0.0), rp(A);
    const double discount = h->search.discount;
    const bool two = h->search.num_players == 2;
    for (size_t i = 0; i < used; ++i) {
        prior[i] = (float)t->child_prior[i];
        if (t->child_visit[i] > 0) {
            // the value term selection reads back: reward + discount * (+/-)(value_sum / visits)   (tree.cuh, tree_backup)
            const double q = t->child_value_sum[i] / (double)t->child_visit[i];
            mval[i] = (double)t->child_reward[i] + discount * (two ? -q : q);
        }
    }
    for (int a = 0; a < A; ++a) rp[a] = t->child_prior[a];
    MZ_CUDA(h, cudaMemcpy(p.visit + base, t->child_visit, used * 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.vsum + base, t->child_value_sum, used * 8, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.mval + base, mval.data(), used * 8, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.reward + base, t->child_reward, used * 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.prior + base, prior.data(), used * 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.expansion + base, t->child_expansion, used * 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.root_prior + (size_t)game * A, rp.data(), A * 8, cudaMemcpyHostToDevice));
    // children of a non-root node: the whole action space (one mask word per game, MZ_MAX_ACTIONS / 32 for |A| > 32)
    const double range[2] = {INFINITY, -INFINITY};
    const int zero = 0;
    if (A > 32) {
        unsigned words[MZ_MAX_ACTIONS / 32];
        for (int j = 0; j < MZ_MAX_ACTIONS / 32; ++j) {
            const int left = A - 32 * j;
            words[j] = left >= 32 ? 0xffffffffu : (left > 0 ? ((1u << left) - 1u) : 0u);
        }
        MZ_CUDA(h, cudaMemcpy(p.legal + (size_t)game * (MZ_MAX_ACTIONS / 32), words, sizeof(words), cudaMemcpyHostToDevice));
    } else {
        const unsigned legal = A >= 32 ? 0xffffffffu : ((1u << A) - 1u);
        MZ_CUDA(h, cudaMemcpy(p.legal + game, &legal, 4, cudaMemcpyHostToDevice));
    }
    MZ_CUDA(h, cudaMemcpy(p.root_visit + game, &t->root_visit, 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.root_vsum + game, &t->root_value_sum, 8, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.root_reward + game, &t->root_reward, 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.range + 2 * (size_t)game, range, 16, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.n_expanded + game, &K, 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.ties + game, &zero, 4, cudaMemcpyHostToDevice));
    MZ_CUDA(h, cudaMemcpy(p.max_depth + game, &zero, 4, cudaMemcpyHostToDevice));
    if (t->hidden) {
        float* dst = p.hidden + (size_t)game * (N + 1) * h->pool_state_elems;
        if (h->net.kind == MZ_NET_RESNET) {
            void* tmp = named_buffer(h, "x.import", (size_t)K * h->hidden_elems * 4);
            if (!tmp) return fail(h, MZ_ENOMEM, "mz_import_tree: out of device memory");
            MZ_CUDA(h, cudaMemcpy(tmp, t->hidden, (size_t)K * h->hidden_elems * 4, cudaMemcpyHostToDevice));
            if (resnet_states_from_nchw(h->res, (const float*)tmp, K, dst, h->stream)) return fail(h, MZ_ECUDA, "mz_import_tree: layout conversion failed");
            MZ_CUDA(h, cudaStreamSynchronize(h->stream));
        } else {
            MZ_CUDA(h, cudaMemcpy(dst, t->hidden, (size_t)K * h->hidden_elems * 4, cudaMemcpyHostToDevice));
        }
    }
    h->imported_expansions = K;
    return MZ_OK;
}

// ------------------------------------------------------------------------------------------
// per-kernel-class device times for bench.py's roofline line (ktimer.h)
extern "C" int mz_kernel_timing(MzHandle* h, int32_t enable) {
    if (!h) return fail(nullptr, MZ_EINVAL, "mz_kernel_timing: null handle");
    kt_enable(enable != 0);
    return MZ_OK;
}

extern "C" int mz_kernel_times(MzHandle* h, double* ms, int64_t* count) {
    if (!h || !ms || !count) return fail(h, MZ_EINVAL, "mz_kernel_times: bad argument");
    cudaSetDevice(h->device);
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < MZ_KERNEL_CLASSES; ++i) { ms[i] = 0.0; count[i] = 0; }
    cudaError_t e = kt_collect(ms, count);
    if (e != cudaSuccess) return fail(h, MZ_ECUDA, std::string("mz_kernel_times: ") + cudaGetErrorString(e));
    return MZ_OK;
}

extern "C" int mz_debug_small_search_plan(int32_t H, int32_t W, int32_t C, int32_t A, int32_t n, int32_t sm_count, int32_t tower_floats,
                                          int32_t heads_floats, int32_t scratch_floats, int32_t cap_channels, int64_t* plan) {
    if (!plan) return 0;
    int P, CO, G, tile, threads, row_stride, board_stride;
    size_t smem;
    if (!small_search_shape(H, W, C, A, n, sm_count, tower_floats, heads_floats, scratch_floats, cap_channels, &P, &CO, &G, &tile, &threads,
                            &smem, &row_stride, &board_stride))
        return 0;
    const int64_t out[8] = {P, CO, G, tile, threads, (int64_t)smem, row_stride, board_stride};
    for (int i = 0; i < 8; ++i) plan[i] = out[i];
    return 1;
}

extern "C" int mz_debug_fc_search_plan(int32_t N, int32_t A, int32_t E, int32_t maxw, int32_t blob_floats, int32_t G, int32_t teacher,
                                       int32_t n, int32_t sm_count, int32_t smem_per_sm, int32_t smem_reserve, int32_t smem_cap,
                                       int32_t regs, int32_t threads, int64_t* plan) {
    FcPlan p;
    if (!plan || smem_per_sm < 0 || smem_reserve < 0 || smem_cap < 0 ||
        !fc_search_plan(N, A, E, maxw, blob_floats, G, teacher != 0, n, sm_count, smem_per_sm, smem_reserve, smem_cap, regs, threads, &p))
        return 0;
    const int64_t out[6] = {p.threads, p.groups, p.ctas_per_sm, p.slots, p.passes, (int64_t)p.smem};
    for (int i = 0; i < 6; ++i) plan[i] = out[i];
    return 1;
}

extern "C" int mz_debug_conv3x3_plan(int32_t n, int32_t cin, int32_t cout, int32_t H, int32_t W, int32_t stride, int64_t* plan) {
    if (!plan) return fail(nullptr, 0, "mz_debug_conv3x3_plan: null plan");
    std::string e;
    if (!resnet_conv_plan(n, cin, cout, H, W, stride, plan, &e)) return fail(nullptr, 0, e);
    return 1;
}

// debug: one conv3x3 through either implementation (host NCHW in / out)
// ------------------------------------------------------------------------------------------
extern "C" int mz_debug_conv3x3(int device, int32_t n, int32_t cin, int32_t cout, int32_t H, int32_t W, int32_t stride, const float* x,
                                const float* w, const float* bias, const float* residual, int32_t relu, int32_t use_tensor_cores,
                                float* out) {
    if (!x || !w || !out || n < 1) return fail(nullptr, MZ_EINVAL, "mz_debug_conv3x3: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_conv3x3: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_conv3x3: device query failed");
    std::string e;
    int rc = resnet_debug_conv(n, cin, cout, H, W, stride, x, w, bias, residual, relu, use_tensor_cores, out, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_conv3x3: " + e);
    return MZ_OK;
}

// debug: one tensor-core tower of one call site of the network (host NCHW in / out)
extern "C" int mz_debug_conv_tower(int device, int32_t n, int32_t H, int32_t W, int32_t mode, int32_t blocks, int32_t site,
                                   int32_t parts, int32_t A, const float* x, const float* w, const float* bias,
                                   const int32_t* action, const int32_t* parent, int32_t pool_stride, float* out,
                                   int64_t* launches, int32_t* saturated) {
    if (!x || !w || !out || !launches) return fail(nullptr, MZ_EINVAL, "mz_debug_conv_tower: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_conv_tower: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_conv_tower: device query failed");
    if (mode != 1 && mode != 2) return fail(nullptr, MZ_EINVAL, "mz_debug_conv_tower: bad shape, site or mode");
    std::string e;
    int rc = resnet_debug_tower(mode == 2 ? TowerRoute::TcX3 : TowerRoute::TcF16, n, 64, 64, H, W, blocks, site, parts, A, x, w,
                                bias, action, parent, pool_stride, out, launches, saturated, nullptr, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_conv_tower: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_small_tower_plan(int32_t n, int32_t in_channels, int32_t C, int32_t H, int32_t W, int32_t blocks,
                                         int32_t stem, int32_t sm_count, int64_t* plan) {
    if (!plan || sm_count < 1) return fail(nullptr, 0, "mz_debug_small_tower_plan: bad argument");
    std::string e;
    if (!resnet_small_tower_plan(n, in_channels, C, H, W, blocks, stem != 0, sm_count, plan, &e))
        return fail(nullptr, 0, "mz_debug_small_tower_plan: " + e);
    return 1;
}

// debug: one fused CUDA-core tower of one call site of the network (host NCHW in / out)
extern "C" int mz_debug_small_tower(int device, int32_t n, int32_t in_channels, int32_t C, int32_t H, int32_t W, int32_t blocks,
                                    int32_t site, int32_t parts, int32_t A, const float* x, const float* w, const float* bias,
                                    const int32_t* action, const int32_t* parent, int32_t pool_stride, float* out, int64_t* plan) {
    if (!x || !w || !out) return fail(nullptr, MZ_EINVAL, "mz_debug_small_tower: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_small_tower: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_small_tower: device query failed");
    std::string e;
    int rc = resnet_debug_tower(TowerRoute::CudaCore, n, in_channels, C, H, W, blocks, site, parts, A, x, w, bias, action, parent,
                                pool_stride, out, nullptr, nullptr, plan, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_small_tower: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_wide_tower_plan(int32_t n, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem, int32_t sm_count,
                                        int64_t* plan) {
    if (!plan || sm_count < 1) return fail(nullptr, 0, "mz_debug_wide_tower_plan: bad argument");
    std::string e;
    if (!resnet_wide_tower_plan(n, C, H, W, blocks, stem != 0, sm_count, plan, &e)) return fail(nullptr, 0, "mz_debug_wide_tower_plan: " + e);
    return 1;
}

// debug: one wide 128-channel tower of one call site of the network (host NCHW in / out)
extern "C" int mz_debug_wide_tower(int device, int32_t n, int32_t H, int32_t W, int32_t blocks, int32_t site, int32_t parts,
                                   int32_t A, const float* x, const float* w, const float* bias, const int32_t* action,
                                   const int32_t* parent, int32_t pool_stride, float* out, int64_t* launches, int32_t* saturated,
                                   int64_t* plan) {
    if (!x || !w || !out || !launches) return fail(nullptr, MZ_EINVAL, "mz_debug_wide_tower: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_wide_tower: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_wide_tower: device query failed");
    std::string e;
    int rc = resnet_debug_tower(TowerRoute::Wide, n, kWideC, kWideC, H, W, blocks, site, parts, A, x, w, bias, action, parent,
                                pool_stride, out, launches, saturated, plan, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_wide_tower: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_wide_pair_tower_plan(int32_t n, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem,
                                             int32_t sm_count, int64_t* plan) {
    if (!plan || sm_count < 1) return fail(nullptr, 0, "mz_debug_wide_pair_tower_plan: bad argument");
    std::string e;
    if (!resnet_wide_tower_plan(n, C, H, W, blocks, stem != 0, sm_count, plan, &e, true))
        return fail(nullptr, 0, "mz_debug_wide_pair_tower_plan: " + e);
    return 1;
}

// debug: one wide 128-channel tower of one call site of the network, each board split across a CTA pair
extern "C" int mz_debug_wide_pair_tower(int device, int32_t n, int32_t H, int32_t W, int32_t blocks, int32_t site, int32_t parts,
                                        int32_t A, const float* x, const float* w, const float* bias, const int32_t* action,
                                        const int32_t* parent, int32_t pool_stride, float* out, int64_t* launches,
                                        int32_t* saturated, int64_t* plan) {
    if (!x || !w || !out || !launches) return fail(nullptr, MZ_EINVAL, "mz_debug_wide_pair_tower: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_wide_pair_tower: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_wide_pair_tower: device query failed");
    std::string e;
    int rc = resnet_debug_tower(TowerRoute::WidePair, n, kWideC, kWideC, H, W, blocks, site, parts, A, x, w, bias, action, parent,
                                pool_stride, out, launches, saturated, plan, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_wide_pair_tower: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_wide256_tower_plan(int32_t n, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem,
                                           int32_t sm_count, int32_t boards, int64_t* plan) {
    if (!plan || sm_count < 1) return fail(nullptr, 0, "mz_debug_wide256_tower_plan: bad argument");
    std::string e;
    if (!resnet_wide256_tower_plan(n, C, H, W, blocks, stem != 0, sm_count, boards, plan, &e))
        return fail(nullptr, 0, "mz_debug_wide256_tower_plan: " + e);
    return 1;
}

// debug: one 256-channel tower of one call site of the network, the output channels split across a CTA pair
extern "C" int mz_debug_wide256_tower(int device, int32_t n, int32_t H, int32_t W, int32_t blocks, int32_t site, int32_t parts,
                                      int32_t A, const float* x, const float* w, const float* bias, const int32_t* action,
                                      const int32_t* parent, int32_t pool_stride, int32_t boards, float* out, int64_t* launches,
                                      int32_t* saturated, int64_t* plan) {
    if (!x || !w || !out || !launches || boards < 0) return fail(nullptr, MZ_EINVAL, "mz_debug_wide256_tower: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_wide256_tower: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_wide256_tower: device query failed");
    std::string e;
    int rc = resnet_debug_tower(TowerRoute::Wide256, n, kWide256C, kWide256C, H, W, blocks, site, parts, A, x, w, bias, action,
                                parent, pool_stride, out, launches, saturated, plan, prop.multiProcessorCount, &e, boards);
    if (rc) return fail(nullptr, rc, "mz_debug_wide256_tower: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_cnn_stem_plan(int32_t n, int32_t in, int32_t C, int32_t H, int32_t W, int32_t sm_count, int64_t* plan) {
    if (!plan) return fail(nullptr, 0, "mz_debug_cnn_stem_plan: null plan");
    std::string e;
    CnnStemPlan p;
    if (!cnn_stem_plan(n, in, C, H, W, sm_count, &p, &e)) return fail(nullptr, 0, "mz_debug_cnn_stem_plan: " + e);
    cnn_stem_plan_export(p, plan);
    return 1;
}

// debug: the DownsampleCNN stem alone (host NCHW in / out)
extern "C" int mz_debug_cnn_stem(int device, int32_t n, int32_t in, int32_t C, int32_t H, int32_t W, const float* x, const float* w1,
                                 const float* b1, const float* w2, const float* b2, float* out, int64_t* plan) {
    if (!x || !w1 || !b1 || !w2 || !b2 || !out || n < 1) return fail(nullptr, MZ_EINVAL, "mz_debug_cnn_stem: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_cnn_stem: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_cnn_stem: device query failed");
    std::string e;
    int rc = cnn_stem_debug(n, in, C, H, W, x, w1, b1, w2, b2, out, plan, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_cnn_stem: " + e);
    return MZ_OK;
}

// debug: the DownSample stem alone (host NCHW in / out)
extern "C" int mz_debug_downsample(int device, int32_t n, int32_t in, int32_t C, int32_t H, int32_t W, const float* x,
                                   const float* w, const float* bias, float* out, float* stages) {
    if (!x || !w || !bias || !out) return fail(nullptr, MZ_EINVAL, "mz_debug_downsample: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_downsample: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_downsample: device query failed");
    std::string e;
    int rc = resnet_debug_downsample(n, in, C, H, W, x, w, bias, out, stages, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_downsample: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_heads_plan(int32_t n, int32_t g0, int32_t C, int32_t H, int32_t W, int32_t site, int32_t layout, int32_t route,
                                   const int32_t* shapes, int32_t sm_count, int64_t* plan) {
    if (!plan || sm_count < 1) return fail(nullptr, 0, "mz_debug_heads_plan: bad argument");
    std::string e;
    if (!resnet_heads_plan(n, g0, C, H, W, site, layout, route, shapes, sm_count, plan, &e)) return fail(nullptr, 0, "mz_debug_heads_plan: " + e);
    return 1;
}

// debug: the heads of one call site of the network (host NCHW in, every output back)
extern "C" int mz_debug_heads(int device, int32_t n, int32_t C, int32_t H, int32_t W, int32_t site, int32_t layout, int32_t route,
                              int32_t parts, const int32_t* shapes, const MzTensor* tensors, int32_t n_tensors, const float* x,
                              int32_t pool_stride, int32_t out_slot, float* logits0, float* logits1, float* scalar, float* rescaled,
                              float* pool, float* state, int64_t* plan) {
    if (!x || (n_tensors > 0 && !tensors)) return fail(nullptr, MZ_EINVAL, "mz_debug_heads: bad argument");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_heads: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_heads: device query failed");
    std::string e;
    int rc = resnet_debug_heads(n, C, H, W, site, layout, route, parts, shapes, tensors, n_tensors, x, pool_stride, out_slot, logits0,
                                logits1, scalar, rescaled, pool, state, plan, prop.multiProcessorCount, &e);
    if (rc) return fail(nullptr, rc, "mz_debug_heads: " + e);
    return MZ_OK;
}

extern "C" int mz_debug_fc_net_plan(const MzNetDesc* net, int32_t obs_elems, int32_t G, int32_t route, int32_t force_split, int32_t n,
                                    int32_t sm_count, int64_t smem_cap, int64_t* plan) {
    if (!net || !plan || smem_cap < 0) return fail(nullptr, 0, "mz_debug_fc_net_plan: bad argument");
    FcNet fc;
    std::vector<float> blob;
    std::string e;
    if (!fc_build_net(*net, obs_elems, nullptr, 0, &fc, &blob, &e) ||
        !fc_debug_plan(fc, G, route, force_split != 0, n, sm_count, (size_t)smem_cap, plan, &e))
        return fail(nullptr, 0, "mz_debug_fc_net_plan: " + e);
    return 1;
}

// debug: one FC network route (host data in, every output back)
extern "C" int mz_debug_fc_net(int device, const MzNetDesc* net, int32_t obs_elems, const MzTensor* tensors, int32_t n_tensors, int32_t G,
                               int32_t route, int32_t force_split, int32_t n, const float* in, const int32_t* action, const int32_t* parent,
                               int32_t pool_stride, int32_t out_slot, float* raw, float* hidden, float* reward_logits, float* value_logits,
                               float* policy_logits, float* prior, float* value, float* reward, float* pool, int64_t* plan) {
    if (!net || !in || !tensors || n_tensors < 1 || !plan || n < 1) return fail(nullptr, MZ_EINVAL, "mz_debug_fc_net: bad argument");
    const bool recurrent = route == MZ_FC_INFER_RECURRENT || route == MZ_FC_INFER_POOL || route == MZ_FC_SEARCH_SIM;
    if (recurrent && !action) return fail(nullptr, MZ_EINVAL, "mz_debug_fc_net: action is null");
    if (route == MZ_FC_INFER_POOL && (!parent || !pool || pool_stride < 1 || out_slot < 0 || out_slot >= pool_stride))
        return fail(nullptr, MZ_EINVAL, "mz_debug_fc_net: bad pool arguments");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_fc_net: no such device");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_fc_net: device query failed");
    FcNet fc;
    std::vector<float> blob;
    std::string e;
    if (!fc_build_net(*net, obs_elems, tensors, n_tensors, &fc, &blob, &e)) return fail(nullptr, MZ_EINVAL, "mz_debug_fc_net: " + e);
    if (!fc_debug_plan(fc, G, route, force_split != 0, n, prop.multiProcessorCount, prop.sharedMemPerBlockOptin, plan, &e))
        return fail(nullptr, MZ_EUNSUPPORTED, "mz_debug_fc_net: " + e);
    const int E = fc.E, A = fc.A, F = fc.F;
    const size_t in_elems = (size_t)n * (recurrent ? E : obs_elems);
    std::vector<void*> bufs;
    cudaError_t err = cudaSuccess;
    // device copy of host data (src) or a buffer of NaN bytes (src == nullptr); nullptr when host is null
    auto dev = [&](const void* host, const void* src, size_t bytes) -> void* {
        if (!host || err != cudaSuccess) return nullptr;
        void* d = nullptr;
        err = cudaMalloc(&d, bytes);
        if (err != cudaSuccess) return nullptr;
        bufs.push_back(d);
        err = src ? cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice) : cudaMemset(d, 0xFF, bytes);
        return d;
    };
    const float* d_blob = (const float*)dev(blob.data(), blob.data(), blob.size() * 4);
    const float* d_in = (const float*)dev(in, route == MZ_FC_INFER_POOL ? nullptr : in, in_elems * 4);
    const int32_t* d_action = (const int32_t*)dev(recurrent ? action : nullptr, action, (size_t)n * 4);
    float* d_raw = (float*)dev(raw, nullptr, (size_t)n * E * 4);
    float* d_hidden = (float*)dev(hidden, nullptr, (size_t)n * E * 4);
    float* d_rl = (float*)dev(reward_logits, nullptr, (size_t)n * F * 4);
    float* d_vl = (float*)dev(value_logits, nullptr, (size_t)n * F * 4);
    float* d_pl = (float*)dev(policy_logits, nullptr, (size_t)n * A * 4);
    float* d_prior = (float*)dev(prior, nullptr, (size_t)n * A * 4);
    float* d_value = (float*)dev(value, nullptr, (size_t)n * 4);
    float* d_reward = (float*)dev(reward, nullptr, (size_t)n * 4);
    const size_t pool_floats = (size_t)n * pool_stride * E;
    std::vector<float> h_pool;
    if (route == MZ_FC_INFER_POOL) {              // NaN bytes everywhere but each sample's parent slot
        h_pool.assign(pool_floats, 0.0f);
        memset(h_pool.data(), 0xFF, pool_floats * 4);
        for (int g = 0; g < n; ++g) {
            if (parent[g] < 0 || parent[g] >= pool_stride) { err = cudaErrorInvalidValue; break; }
            memcpy(h_pool.data() + ((size_t)g * pool_stride + parent[g]) * E, in + (size_t)g * E, (size_t)E * 4);
        }
    }
    float* d_pool = (float*)dev(route == MZ_FC_INFER_POOL ? pool : nullptr, h_pool.data(), pool_floats * 4);
    const int32_t* d_parent = (const int32_t*)dev(route == MZ_FC_INFER_POOL ? parent : nullptr, parent, (size_t)n * 4);
    if (err == cudaSuccess) {
        if (route == MZ_FC_SEARCH_ROOT || route == MZ_FC_SEARCH_SIM) {
            FcDebugArgs a{};
            a.n = n; a.route = route; a.force_split = force_split != 0; a.net = fc; a.blob = d_blob; a.in = d_in; a.action = d_action;
            a.raw = d_raw; a.hidden = d_hidden; a.reward_logits = d_rl; a.value_logits = d_vl; a.policy_logits = d_pl;
            a.prior = d_prior; a.value = d_value; a.reward = d_reward;
            err = launch_fc_debug_net(a, G, plan, 0);
        } else if (route == MZ_FC_INFER_POOL) {
            InferCall c{};
            c.n = n; c.recurrent = 1; c.action = d_action; c.gather_parent = d_parent; c.pool_hidden = d_pool;
            c.pool_stride = pool_stride; c.out_slot = out_slot; c.value_logits = d_vl; c.reward_logits = d_rl;
            c.policy_logits = d_pl; c.hidden = d_hidden; c.value = d_value; c.reward = d_reward;
            err = launch_fc_inference_pool(fc, d_blob, c, G, prop.multiProcessorCount, prop.sharedMemPerBlockOptin, 0);
        } else {
            FcInferArgs a{};
            a.n = n; a.recurrent = recurrent; a.net = fc; a.blob = d_blob; a.in = d_in; a.action = d_action;
            a.value_logits = d_vl; a.reward_logits = d_rl; a.policy_logits = d_pl; a.hidden = d_hidden; a.value = d_value;
            a.reward = d_reward;
            err = launch_fc_inference(a, G, prop.multiProcessorCount, prop.sharedMemPerBlockOptin, 0);
        }
    }
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    const struct { void* host; const void* d; size_t bytes; } back[] = {
        {raw, d_raw, (size_t)n * E * 4}, {hidden, d_hidden, (size_t)n * E * 4}, {reward_logits, d_rl, (size_t)n * F * 4},
        {value_logits, d_vl, (size_t)n * F * 4}, {policy_logits, d_pl, (size_t)n * A * 4}, {prior, d_prior, (size_t)n * A * 4},
        {value, d_value, (size_t)n * 4}, {reward, d_reward, (size_t)n * 4}, {pool, d_pool, pool_floats * 4}};
    for (const auto& b : back)
        if (err == cudaSuccess && b.host && b.d) err = cudaMemcpy(b.host, b.d, b.bytes, cudaMemcpyDeviceToHost);
    for (void* d : bufs) cudaFree(d);
    if (err != cudaSuccess) return fail(nullptr, MZ_ECUDA, std::string("mz_debug_fc_net: ") + cudaGetErrorString(err));
    return MZ_OK;
}
