/*
 * mzb200 - C ABI of the H100-native self-play search library (libmzb200.so).
 *
 * The reference (werner-duvaud/muzero-general) is pure Python and has no FFI; the drop-in
 * boundary is therefore the set of Python call sites listed next to each entry point below
 * (file:line in the reference).  A maintainer binds these symbols with ctypes
 * (see INTEGRATION.md and muzero_general_b200/_lib.py); nothing here mentions torch.
 *
 * Conventions
 *   - every function returns 0 on success, a negative MZ_E* code on failure; the message is
 *     available from mz_last_error(handle) (or mz_last_error(NULL) for mz_create failures);
 *     the library never aborts the process;
 *   - the caller owns every buffer passed in; the library borrows it for the duration of the
 *     call.  `mem` says whether the IO pointers of that call are HOST or DEVICE pointers
 *     (device = the handle's device).  Host buffers are staged through library-owned pinned
 *     memory, copies included in the call;
 *   - a handle is NOT thread-safe: one host thread per handle, one handle per GPU process
 *     (mirrors the reference's one-thread-per-actor model, self_play.py:11-29);
 *   - all library-owned scratch (node pool, hidden-state pool, staging) is allocated in
 *     mz_create, sized from max_games, num_simulations, action_space and the net shape.
 */
#ifndef MZB200_H
#define MZB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MZ_ABI_VERSION 2
#define MZ_MAX_LAYERS 8          /* hidden layers per MLP head */
#define MZ_MAX_ACTIONS 256       /* |action_space| supported by the tree kernels (one lane per action up to 32; above,
                                    one warp per game with four actions per lane up to 128 and eight up to 256:
                                    csrc/tree_wide.cu).  256 is the ceiling of this ABI version: MzTrace.actions is
                                    uint8_t, so action ids 0..255 are what a trace can record */

enum { MZ_OK = 0, MZ_EINVAL = -1, MZ_ECUDA = -2, MZ_EUNSUPPORTED = -3, MZ_ESTATE = -4, MZ_ENOMEM = -5 };
enum { MZ_NET_FC = 0, MZ_NET_RESNET = 1 };
enum { MZ_MEM_HOST = 0, MZ_MEM_DEVICE = 1 };

/* Shape of the networks built by models.MuZeroNetwork(config)  (models.py:7-41). */
typedef struct MzNetDesc {
    int32_t kind;                 /* MZ_NET_FC (models.py:80-195) or MZ_NET_RESNET (models.py:436-623) */
    int32_t obs_c, obs_h, obs_w;  /* stacked input: C*(s+1)+s channels, H, W (self_play.py:513-550) */
    int32_t action_space;         /* len(config.action_space); actions are 0..A-1 */
    int32_t support_size;         /* config.support_size; heads emit 2S+1 logits */
    /* fully connected */
    int32_t encoding;
    int32_t n_fc_representation, fc_representation[MZ_MAX_LAYERS];
    int32_t n_fc_dynamics, fc_dynamics[MZ_MAX_LAYERS];
    int32_t n_fc_reward, fc_reward[MZ_MAX_LAYERS];
    int32_t n_fc_value, fc_value[MZ_MAX_LAYERS];
    int32_t n_fc_policy, fc_policy[MZ_MAX_LAYERS];
    /* residual */
    int32_t blocks, channels;
    int32_t reduced_reward, reduced_value, reduced_policy;
    int32_t n_res_fc_reward, res_fc_reward[MZ_MAX_LAYERS];
    int32_t n_res_fc_value, res_fc_value[MZ_MAX_LAYERS];
    int32_t n_res_fc_policy, res_fc_policy[MZ_MAX_LAYERS];
    int32_t downsample;           /* 0 = none, 1 = "resnet" (models.py:233-275), 2 = "CNN" (models.py:278-297) */
} MzNetDesc;

/* The MuZeroConfig attributes MCTS reads (self_play.py:249-430). */
typedef struct MzSearchDesc {
    int32_t max_games;            /* capacity B: games searched in lockstep by one call */
    int32_t num_simulations;      /* config.num_simulations */
    int32_t num_players;          /* len(config.players); 1 or 2 (self_play.py:411-430) */
    int32_t extra_expansions;     /* node-pool room beyond num_simulations + 1 expansions per game, for searches that
                                     continue from an imported tree (override_root_with, self_play.py:275-277); the
                                     three tables below then have num_simulations + extra_expansions + 2 entries (per side) */
    double discount;              /* config.discount */
    double pb_c_base, pb_c_init;  /* self_play.py:384-390 */
    double root_dirichlet_alpha;  /* used only when noise is generated on the device */
    double root_exploration_fraction; /* self_play.py:476 */
    uint64_t seed;                /* key of the counter-based tie-break / noise stream */
    /* log((n+base+1)/base)+init and sqrt(n) for n = 0..num_simulations+1, computed by the
     * caller with the host language's libm so the device reproduces math.log / math.sqrt
     * (self_play.py:385-390) exactly.  NULL: the library computes them with C log()/sqrt(). */
    const double* pb_c_table;
    const double* sqrt_table;
    /* optional [(N+2) x (N+2)]: ucb_table[n_p*(N+2) + n_c] = pb_c_table[n_p] * (sqrt_table[n_p] / (n_c + 1)), i.e. the
     * exploration factor of self_play.py:384-390 with its two roundings, evaluated by the caller; saves two fp64
     * operations (one division) per child per tree level on the device.  NULL: computed on the device. */
    const double* ucb_table;
} MzSearchDesc;

/* One named tensor of the reference state_dict (models.py:69-73), fp32 host memory. */
typedef struct MzTensor {
    const char* name;             /* e.g. "dynamics_encoded_state_network.module.0.weight" */
    const float* data;
    int64_t numel;
} MzTensor;

/* Optional per-simulation record of what the device did (student forcing, SURVEY.md 8c). */
typedef struct MzTrace {
    int32_t max_depth;            /* D: entries kept per path */
    int32_t reserved;
    int32_t* depth;               /* [n, N]      number of select_child calls of simulation i */
    uint8_t* actions;             /* [n, N, D]   actions chosen root->leaf; 0 past the path's depth (host buffers; a
                                                  device buffer keeps what it held there) */
    float* value;                 /* [n, N]      scalarised value of the expanded leaf */
    float* reward;                /* [n, N]      scalarised reward of the expanded leaf */
    float* priors;                /* [n, N, A]   fp32 softmax priors of the expanded leaf */
    float* root_priors_raw;       /* [n, A]      root priors before noise (0 for illegal) */
    float* root_reward;           /* [n] */
    double* noise;                /* [n, A]      Dirichlet noise mixed into the root priors (given or device-drawn) */
} MzTrace;

/* Teacher forcing: bypass the networks, feed the tree these per-simulation outputs instead. */
typedef struct MzTeacher {
    const float* root_value;      /* [n] */
    const float* root_reward;     /* [n] */
    const float* root_priors;     /* [n, A] by action id (illegal entries ignored) */
    const float* value;           /* [n, N] */
    const float* reward;          /* [n, N] */
    const float* priors;          /* [n, N, A] */
} MzTeacher;

/* Arguments of one batched MCTS.run (self_play.py:260-361) over n games. */
typedef struct MzSearchIO {
    int32_t n_games;              /* <= max_games */
    int32_t mem;                  /* MZ_MEM_HOST or MZ_MEM_DEVICE for every pointer below */
    /* inputs */
    const float* obs;             /* [n, obs_c*obs_h*obs_w] fp32 (torch.tensor(obs).float(), self_play.py:281-282) */
    const uint8_t* legal_mask;    /* [n, A] non-zero = legal (self_play.py:296-308); NULL = all legal */
    const int32_t* to_play;       /* [n] game.to_play(); NULL = 0 */
    int32_t add_exploration_noise;/* self_play.py:310-314 */
    int32_t flags;                /* MZ_FLAG_* */
    const double* noise;          /* [n, A] Dirichlet draw by action id (host draws); NULL = drawn on the device
                                     (Philox + Marsaglia-Tsang gamma, root_dirichlet_alpha) */
    const int32_t* first_index;   /* [n] index into the legal list picked at the first simulation's
                                     all-way tie (self_play.py:371); NULL = device Philox */
    const int64_t* game_id;       /* [n] global game ids keying the Philox stream; NULL = 0..n-1 */
    const int32_t* move_index;    /* [n] move number keying the Philox stream; NULL = 0 */
    /* outputs (any may be NULL) */
    int32_t* visit_counts;        /* [n, A] child.visit_count by action id, 0 if illegal */
    double* root_value;           /* [n] root.value() (self_play.py:509) */
    float* root_predicted_value;  /* [n] mcts_info["root_predicted_value"] */
    int32_t* max_tree_depth;      /* [n] mcts_info["max_tree_depth"] */
    int32_t* tie_count;           /* [n] exact UCB ties met after the first simulation */
    double* root_priors;          /* [n, A] root priors after noise */
    double* value_range;          /* [n, 2] MinMaxStats minimum, maximum */
    const MzTeacher* teacher;     /* NULL = use the networks */
    const MzTrace* trace;         /* NULL = no trace */
} MzSearchIO;

/* Arguments of mz_search_device: the search of MzSearchIO with mem = MZ_MEM_DEVICE, flags = 0 and neither teacher nor
 * trace.  Every pointer is device memory with the meaning of the MzSearchIO field of the same name. */
typedef struct MzDeviceSearchIO {
    int32_t n_games;              /* <= max_games */
    int32_t add_exploration_noise;
    const float* obs;             /* required */
    const double* noise;
    const int64_t* game_id;
    const int32_t* move_index;
    const uint8_t* legal_mask;
    const int32_t* to_play;
    const int32_t* first_index;
    int32_t* visit_counts;
    double* root_value;
    float* root_predicted_value;
    int32_t* max_tree_depth;
    int32_t* tie_count;
    double* root_priors;
    double* value_range;
    double device_ms;             /* out: mz_last_search_ms of this call */
} MzDeviceSearchIO;

#define MZ_FLAG_KEEP_TREE 1       /* leave the full tree in the HBM node pool for mz_export_tree */
#define MZ_FLAG_STEPWISE  2       /* force the generic select/infer/expand+backup pipeline */
#define MZ_FLAG_CONTINUE  4       /* MCTS.run(..., override_root_with=node), self_play.py:275-277: no root inference; the
                                     search runs num_simulations more simulations on the tree mz_import_tree put into the
                                     pool (n_games must be 1; fresh MinMaxStats; the root noise is mixed into the
                                     imported root priors).  obs is ignored. */

/* Full tree of one game after a search with MZ_FLAG_KEEP_TREE (host pointers). Slot layout:
 * expansion e (0 = root, e = i+1 for simulation i) owns child slots [e*A, e*A+A). */
typedef struct MzTreeExport {
    int32_t n_expansions;         /* out */
    int32_t* child_visit;         /* [(N+1)*A] */
    double* child_value_sum;      /* [(N+1)*A] */
    float* child_reward;          /* [(N+1)*A] */
    double* child_prior;          /* [(N+1)*A] */
    int32_t* child_expansion;     /* [(N+1)*A] expansion id of the child, -1 if not expanded */
    float* hidden;                /* [(N+1), hidden_elems] or NULL */
    int32_t root_visit;           /* out */
    double root_value_sum;        /* out */
    float root_reward;            /* out: reward of the root node (-0.0 for a fresh root; the child's reward after an import) */
    int32_t reserved;
} MzTreeExport;

/* Results of a batched network call, all DEVICE or all HOST per `mem`; any pointer may be NULL. */
typedef struct MzInferenceOut {
    float* value_logits;          /* [n, 2S+1] */
    float* reward_logits;         /* [n, 2S+1] */
    float* policy_logits;         /* [n, A] */
    float* hidden;                /* [n, hidden_elems] (rescaled state) */
    float* value;                 /* [n] support_to_scalar(value_logits)  (models.py:645-666) */
    float* reward;                /* [n] support_to_scalar(reward_logits) */
} MzInferenceOut;

typedef struct MzHandle MzHandle;

/* replaces SelfPlay.__init__ model construction (self_play.py:25-29) + MCTS(config) (self_play.py:257-258) */
int mz_create(const MzNetDesc* net, const MzSearchDesc* search, int device, MzHandle** out);
int mz_destroy(MzHandle* h);
const char* mz_last_error(const MzHandle* h);
int mz_abi_version(void);

/* replaces model.set_weights(state_dict) (models.py:72-73, self_play.py:27,37) */
int mz_load_weights(MzHandle* h, const MzTensor* tensors, int32_t n_tensors);

/* replaces MCTS.run for a batch of games (self_play.py:260-361; called from self_play.py:144-150) */
int mz_search(MzHandle* h, const MzSearchIO* io);
/* The same search on device buffers in two calls, with less host work: mz_search_device enqueues it and returns (no
 * staging or debug outputs; the fused FC route launches the kernel its handle prepared for the last n_games and A/B
 * switches it saw), mz_search_device_wait waits for it and sets io->device_ms.  The outputs are complete after the wait;
 * work the caller does in between overlaps the search.  Every mz_search_device must be followed by its wait before the
 * next call on the handle.  Results are mz_search's. */
int mz_search_device(MzHandle* h, MzDeviceSearchIO* io);
int mz_search_device_wait(MzHandle* h, MzDeviceSearchIO* io);

/* replaces model.initial_inference / recurrent_inference (models.py:172-195, 601-623) */
int mz_initial_inference(MzHandle* h, int32_t n, int32_t mem, const float* obs, const MzInferenceOut* out);
int mz_recurrent_inference(MzHandle* h, int32_t n, int32_t mem, const float* hidden, const int32_t* action,
                           const MzInferenceOut* out);

/* Arguments of mz_reanalyse_values: the fresh root values of every position of n games (Reanalyse, replay_buffer.py:
 * 345-366).  `mem` says where frames, actions and values live; the offsets and positions are HOST arrays (the library
 * plans its chunks from them).  Game g owns frame rows [frame_offsets[g], frame_offsets[g + 1]) (its observation_history)
 * and entries [action_offsets[g], action_offsets[g + 1]) of actions (its action_history, leading 0 included); its
 * positions are i = 0 .. positions[g] - 1 (len(root_values)).  The stack depth s is the handle's: obs_elems =
 * O + s * (O + H * W) with O = frame_elems and H x W the handle's obs_h x obs_w. */
typedef struct MzReanalyseIO {
    int32_t n_games;
    int32_t mem;                  /* MZ_MEM_HOST or MZ_MEM_DEVICE for frames, actions and values */
    int32_t stacked_observations; /* the caller's s: must be the handle's */
    int32_t reserved;
    int64_t frame_elems;          /* O: floats per frame (the environment's C x H x W observation) */
    const float* frames;          /* [F][O] fp32, every game's observation_history back to back */
    const int64_t* frame_offsets; /* [n + 1] host, non-negative, non-decreasing */
    const int32_t* actions;       /* [action_offsets[n]] every game's action_history back to back, each in [0, A) */
    const int64_t* action_offsets;/* [n + 1] host, non-negative, non-decreasing */
    const int64_t* positions;     /* [n] host: T_g, 0 <= T_g <= frames of game g, and T_g <= actions of game g */
    float* values;                /* [sum T_g] out: support_to_scalar(initial_inference(stacked input)[0]), game order */
} MzReanalyseIO;

/* replaces the stacked-observation gathering and model.initial_inference of Reanalyse (replay_buffer.py:345-366) for a
 * batch of games: the positions, in game order, are cut into chunks of at most max_games (a chunk may span many games
 * or cut through one); per chunk a kernel builds each position's stacked input, GameHistory.get_stacked_observations(
 * i, s, A) (self_play.py:304-315), in the representation's input workspace and the network of mz_initial_inference
 * runs on it (its route, its range guard).  With host memory each chunk's frame rows (the positions' rows and the s
 * before the first) are staged through two pinned buffers, the next chunk's upload overlapping the current chunk's
 * network; device memory is read in place.  The staging buffers are allocated by the first call and kept with the
 * handle (a larger frame_elems or s grows them).  Beyond mz_create's allocations the call takes at most
 * 2 x ((max_games + s) x (O + 1) x 4 + max_games x 20) bytes of device memory (and as much pinned host memory with host
 * frames), whatever the games' lengths.  Refused with MZ_EINVAL, before anything is written: stacked_observations other
 * than the handle's, a frame_elems that with it does not give obs_elems (the message names the s the handle implies for
 * that O), negative or decreasing offsets, a T_g outside [0, frames of g] or above the game's actions, an action outside
 * [0, A). */
int mz_reanalyse_values(MzHandle* h, const MzReanalyseIO* io);
/* Debug / parity: the stacked inputs chunk `chunk` of mz_reanalyse_values(h, io) builds, without the network: out (HOST)
 * receives [n_c][obs_elems] floats, n_c = the chunk's positions; io->values is not used.  The refusals of
 * mz_reanalyse_values, and MZ_EINVAL for a chunk beyond the call's. */
int mz_debug_reanalyse_stack(MzHandle* h, const MzReanalyseIO* io, int32_t chunk, float* out);

/* Arguments of mz_reanalyse_search: the self-play search re-run at every position of n games (the MuZero paper's
 * Reanalyze).  The positions are games' as in mz_reanalyse_values (games->values is not used); `games->mem` also says
 * where legal_mask, to_play and the outputs live.  Position i of game g is searched as MCTS.run(model,
 * get_stacked_observations(i, s, A), legal actions, to_play, add_exploration_noise) with the Philox streams keyed by
 * (seed, game_id[g], move index i), so a position searched with its self-play game id reproduces that move's search. */
typedef struct MzReanalyseSearchIO {
    const MzReanalyseIO* games;   /* frames, actions, offsets, positions, mem, s and O, as mz_reanalyse_values takes them */
    const uint8_t* legal_mask;    /* [sum T_g][A] non-zero = legal, game order; NULL = all legal */
    const int32_t* to_play;       /* [sum T_g] to_play_history[i], each in [0, num_players); NULL = 0 */
    const int64_t* game_id;       /* [n] HOST: the Philox game id of each game; NULL = 0 .. n - 1 */
    int32_t add_exploration_noise;/* self_play.py:310-314 (the root noise is drawn on the device) */
    int32_t reserved;
    int32_t* visit_counts;        /* [sum T_g][A] out: child.visit_count by action id, 0 if illegal, game order */
    double* root_value;           /* [sum T_g] out: root.value(), game order; may be NULL */
} MzReanalyseSearchIO;

/* Fresh policy targets for Reanalyse: per chunk of at most max_games positions, the stack of mz_reanalyse_values, then a
 * kernel writes each position's legal row, to_play, game id and move index into the search's input arena and the search
 * of mz_search runs on them (the same route: fused FC, fused small search, step-wise towers, the x3 range guard).  With
 * host memory the legal rows and to_play travel with the chunk's frames through the two pinned staging buffers, and the
 * results come back through the handle's pinned output arena while the next chunk searches; device memory is read and
 * written in place.  Beyond mz_create's allocations the call takes at most 2 x ((max_games + s) x (O + 1) x 4 +
 * max_games x (32 + A)) bytes of device memory (and as much pinned host memory with host memory), plus 256-byte
 * alignment per staged array, whatever the games' lengths.  With device memory the checks below read the legal masks
and to_play on the host: sum T_g x (A + 4) bytes of host memory for the duration of the call.  Refused with MZ_EINVAL, before anything is written: every
 * refusal of mz_reanalyse_values, visit_counts NULL with positions to search, a position without a legal action, a to_play
 * outside [0, num_players).  MZ_ESTATE: a handle created with num_simulations = 0. */
int mz_reanalyse_search(MzHandle* h, const MzReanalyseSearchIO* io);

/* Node graph access for callers that walk the tree (self_play.py:229-232,499-509; diagnose_model.py:164,222-255) */
int mz_export_tree(MzHandle* h, int32_t game, MzTreeExport* out);
/* The inverse: seed game `game`'s tree in the pool from host arrays in the same layout (n_expansions, root_visit,
 * root_value_sum, root_reward are inputs; hidden = [n_expansions, hidden_elems] dense states, required unless the
 * search is teacher-forced).  Used by MCTS.run(override_root_with=...) followed by mz_search(MZ_FLAG_CONTINUE). */
int mz_import_tree(MzHandle* h, int32_t game, const MzTreeExport* tree);

/* sizes derived from the descriptors */
int64_t mz_hidden_elems(const MzHandle* h);
int64_t mz_obs_elems(const MzHandle* h);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t mz_launch_count(const MzHandle* h);
/* parallel branches of the CUDA graph the step-wise search is replayed from: the simulations of disjoint game ranges
 * overlap (towers of one range with the heads / tree steps of the others); 1 = a single chain.  MZ_PARTS=1..4 overrides. */
int32_t mz_graph_partitions(const MzHandle* h);
/* device time of the search kernels of the last mz_search call, ms (CUDA events on the library stream) */
double mz_last_search_ms(const MzHandle* h);
/* host side of the last search call: out[4] = CLOCK_MONOTONIC ns (Python's time.perf_counter_ns) at its entry, when the
 * search was enqueued, when the stream synchronisation returned, and at its return (scripts/search_host_split.py) */
int mz_debug_host_split(const MzHandle* h, int64_t* out);
/* shape of the handle's last launch of the fused FC search kernel (csrc/fc_search.cu): returns 1 and fills info[5] =
 * {grid, threads per CTA, lanes per game, shared-memory bytes per CTA, resident CTAs per SM}, or 0 before the first one */
int mz_fc_last_launch(const MzHandle* h, int64_t* info);
/* the fused FC launch the handle keeps for its next search: returns 1 and fills info[7] = {games, lanes per game, fixed
 * CTA size (0 = planned), MZ_FC_GENERIC=1, MZ_FC_SELECT_LEVELS=1, tree levels per selection round, 1 = the fixed-shape
 * network instantiation}, or 0 when there is none (no fused launch yet, or the weights were loaded since) */
int mz_debug_fc_prepared(const MzHandle* h, int64_t* info);

/* Per-kernel-class device timing for the roofline line of bench.py.  While enabled (process-wide), the step-wise
 * pipeline runs launch by launch with a CUDA event pair around every kernel instead of replaying its CUDA graph.
 * mz_kernel_times synchronises and returns the accumulated milliseconds / launch counts since the last call:
 * [0] tree_step_kernel, [1] conv_tower_tc_kernel (wgmma towers, resident or streaming), [2] heads_kernel,
 * [3] conv3x3_kernel (CUDA cores, one conv per launch), [4] other, [5] small_tower_kernel (fused CUDA-core towers),
 * [6] small_search_kernel (small residual networks: all simulations of a search in one launch). */
#define MZ_KERNEL_CLASSES 7
int mz_kernel_timing(MzHandle* h, int32_t enable);
int mz_kernel_times(MzHandle* h, double* ms, int64_t* count);

/* Debug / tests (host only, no device needed): launch plan of the fused small-network search (csrc/small_search.cu) for a
 * hidden board H x W x C, |A| actions, n games on sm_count SMs, with tower_floats + heads_floats of weights and scratch_floats
 * of per-warp scratch in shared memory and cap_channels channels per activation buffer.  Returns 1 and fills
 * plan[8] = {P, CO, G, games per CTA, threads per CTA, shared-memory bytes, row stride, board stride}, or 0 when the shape
 * is not handled (the step-wise pipeline is used then). */
int mz_debug_small_search_plan(int32_t H, int32_t W, int32_t C, int32_t A, int32_t n, int32_t sm_count, int32_t tower_floats,
                               int32_t heads_floats, int32_t scratch_floats, int32_t cap_channels, int64_t* plan);

/* Debug / tests (host only, no device needed): CTA size of the fused FC search (csrc/fc_search.cu::fc_search_plan) for
 * N simulations, |A| actions, encoding E, widest layer maxw, blob_floats floats of weights, G lanes per game, the teacher-
 * forced kernel or not, n games on sm_count SMs with smem_per_sm bytes of shared memory per SM, smem_reserve of it taken
 * per CTA, smem_cap bytes at most per CTA and regs registers per thread; threads = 0 picks the CTA size (the fewest
 * passes, then the smallest CTA), else plans that size.  Returns 1 and fills plan[6] = {threads per CTA, games per CTA,
 * CTAs per SM, resident games, passes, shared-memory bytes per CTA}, or 0 when a game does not fit (the search then
 * runs step by step). */
int mz_debug_fc_search_plan(int32_t N, int32_t A, int32_t E, int32_t maxw, int32_t blob_floats, int32_t G, int32_t teacher,
                            int32_t n, int32_t sm_count, int32_t smem_per_sm, int32_t smem_reserve, int32_t smem_cap,
                            int32_t regs, int32_t threads, int64_t* plan);

/* Debug / tests (host only, no device needed): launch plan of the CUDA-core conv3x3 kernel (csrc/resnet.cu) for n boards of
 * cin x H x W -> cout channels at stride 1 or 2.  Returns 1 and fills plan[12] = {P (pixels per thread), stride,
 * MAX_ITEMS (accumulator tiles per thread), row bands, rows per band, boards per CTA, cin chunk, grid x, grid y (cout
 * tiles), grid z, shared-memory bytes, cout tile (64, or fewer channels when one output row of 64 exceeds a CTA's
 * items)}, or 0 with the reason in mz_last_error(NULL) when the shape cannot be launched.  mz_create refuses a net with
 * such a conv. */
int mz_debug_conv3x3_plan(int32_t n, int32_t cin, int32_t cout, int32_t H, int32_t W, int32_t stride, int64_t* plan);

/* Debug / parity: one conv3x3 (cin -> cout, stride 1 or 2, pad 1; models.py:206-209) with optional bias, residual and
 * ReLU on host NCHW fp32 data, through the CUDA-core kernel (use_tensor_cores = 0; cout a multiple of 4) or the wgmma
 * implicit GEMM (64 -> 64, stride 1, H <= 6, W <= 7, else MZ_EUNSUPPORTED): 1 = fp16 operands, 2 = split fp16 operands
 * with three partial products (fp32-grade, the default of the search path).  x is [n][cin][H][W], w is [cout][cin][3][3]
 * as in the reference state_dict, bias [cout], residual and out [n][cout][Ho][Wo] with Ho = (H - 1) / stride + 1 (same
 * for Wo).  The device output is filled with NaN before the launch, so an element the kernel does not write reads NaN. */
int mz_debug_conv3x3(int device, int32_t n, int32_t cin, int32_t cout, int32_t H, int32_t W, int32_t stride, const float* x,
                     const float* w, const float* bias, const float* residual, int32_t relu, int32_t use_tensor_cores, float* out);

/* Call sites of the towers (site argument of mz_debug_conv_tower and mz_debug_small_tower) */
#define MZ_TOWER_REPRESENTATION 0   /* input in a workspace, reusable once read; no stem */
#define MZ_TOWER_DYNAMICS 1         /* plain recurrent call: input converted into a workspace; stem with the action plane */
#define MZ_TOWER_DYNAMICS_POOL 2    /* in search: input gathered from the hidden-state pool (read only); stem with the action plane */
#define MZ_TOWER_PREDICTION 3       /* input in the rescaled-state scratch buffer, reusable; no stem */

/* Debug / parity: one whole tensor-core tower (models.py:213-229 without BN: [stem conv +] `blocks` residual blocks, every
 * conv with bias and ReLU) of one call site of the network on host NCHW fp32 data, through the launch packing and the
 * kernels the network runs (mode 1 = fp16 operands, 2 = x3).  H <= 6, W <= 7.  x is [n][64][H][W]; w holds every conv's
 * [cout 64][cin][3][3] back to back (the dynamics stem first, cin = 65: channel 64 is the action plane action[g] / A), bias
 * [convs][64] (or NULL); action [n] in [0, A) for the dynamics sites; at MZ_TOWER_DYNAMICS_POOL game g's input sits in slot
 * parent[g] of its pool_stride slots, the other slots hold NaN, and `parts` (x3 only, 1..4) runs the games in the ranges of
 * the partitioned replay.  Workspaces and output start as NaN.  out is [n][64][H][W]; *launches gets the number of kernel
 * launches of the tower and *saturated the x3 range-guard count (stored activations beyond the fp16 range). */
int mz_debug_conv_tower(int device, int32_t n, int32_t H, int32_t W, int32_t mode, int32_t blocks, int32_t site, int32_t parts,
                        int32_t A, const float* x, const float* w, const float* bias, const int32_t* action, const int32_t* parent,
                        int32_t pool_stride, float* out, int64_t* launches, int32_t* saturated);

/* Launch plan of the fused CUDA-core tower (host only): n boards of H x W through [a stem conv reading in_channels planes,
 * C + 1 for the dynamics stem with its action plane, if stem] + `blocks` residual blocks of C channels.  Fills plan[6] =
 * {P pixels per thread, CO output channels per thread, boards per CTA, threads per CTA, persistent grid, dynamic shared-memory
 * bytes} and returns 1; returns 0 with the reason in mz_last_error(NULL) when the fused tower refuses the shape (the network
 * then runs one conv3x3 launch per conv). */
int mz_debug_small_tower_plan(int32_t n, int32_t in_channels, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem,
                              int32_t sm_count, int64_t* plan);

/* Debug / parity: one fused CUDA-core tower (models.py:206-231 without BN: [stem conv +] `blocks` residual blocks, every conv
 * with bias and ReLU, the residual added before the second ReLU of a block) of one call site of resnet_inference on host NCHW
 * fp32 data, through the helper the network calls.  MZ_TOWER_REPRESENTATION: stem from x [n][in_channels][H][W];
 * MZ_TOWER_DYNAMICS: stem of C + 1 planes, channel C the action plane action[g] / A, x [n][C][H][W] dense;
 * MZ_TOWER_DYNAMICS_POOL: the same with game g's input in slot parent[g] of its pool_stride slots, the other slots NaN, and
 * `parts` (1..4) runs the games in the ranges of the partitioned replay; MZ_TOWER_PREDICTION: no stem, blocks >= 1
 * (in_channels is C at every site but the representation).  w holds every conv's [C][cin][3][3] back to back, bias [convs][C]
 * (or NULL).  The output starts as NaN.  out is [n][C][H][W]; plan (or NULL) gets the plan of the launch as
 * mz_debug_small_tower_plan fills it (of the first range when partitioned).  MZ_EUNSUPPORTED when the fused tower refuses the
 * shape. */
int mz_debug_small_tower(int device, int32_t n, int32_t in_channels, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t site,
                         int32_t parts, int32_t A, const float* x, const float* w, const float* bias, const int32_t* action,
                         const int32_t* parent, int32_t pool_stride, float* out, int64_t* plan);

/* Launch plan of the wide tower (host only; the route MZ_TC_WIDE=1 opts 128-channel nets into): n boards of C x H x W
 * through [a stem conv, C + 1 planes with the action plane, if stem] + `blocks` residual blocks as x3 tensor-core MMAs, one
 * board per CTA.  Fills plan[9] = {M-tiles of 64 board rows, threads per CTA, dynamic shared-memory bytes, weight ring
 * stages, layers, CTAs per SM, boards per wave, launches per tower call, registers per thread assumed} and returns 1;
 * returns 0 with the reason in mz_last_error(NULL) when the wide towers refuse the shape (C != 128, a board beyond the
 * shared-memory or M-tile budget, more than 10 blocks): the network then keeps the CUDA-core towers. */
int mz_debug_wide_tower_plan(int32_t n, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem, int32_t sm_count,
                             int64_t* plan);

/* Debug / parity: one wide tower (128 channels, models.py:206-231 without BN: [stem conv +] `blocks` residual blocks, every
 * conv with bias and ReLU) of one call site of resnet_inference on host NCHW fp32 data, through the helper and the weight
 * packing the network uses.  x is [n][128][H][W] (at MZ_TOWER_REPRESENTATION the output of the CUDA-core stem); w holds
 * every conv's [128][cin][3][3] back to back (the dynamics stem first, cin = 129: channel 128 is the action plane
 * action[g] / A), bias [convs][128] (or NULL); at MZ_TOWER_DYNAMICS_POOL game g's input sits in slot parent[g] of its
 * pool_stride slots, the other slots hold NaN, and `parts` (1..4) runs the games in the ranges of the partitioned replay.
 * The output starts as NaN.  out is [n][128][H][W]; *launches gets the kernel launches, *saturated the range-guard count
 * (activations read or stored beyond the fp16 range) and plan (or NULL) the plan of the first range as
 * mz_debug_wide_tower_plan fills it.  MZ_EUNSUPPORTED when the wide towers refuse the shape. */
int mz_debug_wide_tower(int device, int32_t n, int32_t H, int32_t W, int32_t blocks, int32_t site, int32_t parts, int32_t A,
                        const float* x, const float* w, const float* bias, const int32_t* action, const int32_t* parent,
                        int32_t pool_stride, float* out, int64_t* launches, int32_t* saturated, int64_t* plan);

/* Launch plan of the wide tower on CTA pairs (host only; the route MZ_TC_WIDE=2 adds for boards the one-CTA plan refuses,
 * e.g. 15 x 15 and 16 x 16): each board split across a cluster of two CTAs, CTA 0 taking rows [0, ceil(H / 2)) and CTA 1
 * the rest, the boundary rows exchanged through distributed shared memory after every layer.  Same arguments as
 * mz_debug_wide_tower_plan.  Fills plan[9] = {board rows of CTA 0, M-tiles per CTA, threads per CTA, dynamic shared-memory
 * bytes per CTA, weight ring stages, layers, boards (CTA pairs) per wave as planned (CTAs per SM x SMs / 2), launches per
 * tower call, registers per thread assumed} and returns 1; returns 0 with the reason in mz_last_error(NULL) when the pair
 * refuses the shape (C != 128, H < 2, a half beyond the shared-memory or M-tile budget, more than 10 blocks).  It accepts
 * every board the one-CTA plan accepts with H >= 2. */
int mz_debug_wide_pair_tower_plan(int32_t n, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem, int32_t sm_count,
                                  int64_t* plan);

/* Debug / parity: mz_debug_wide_tower with every board split across a CTA pair: the same arguments, data and outputs (plan
 * as mz_debug_wide_pair_tower_plan fills it).  It always runs the pair kernel on a shape its planner accepts, including
 * boards one CTA could hold.  MZ_EUNSUPPORTED when the pair refuses the shape. */
int mz_debug_wide_pair_tower(int device, int32_t n, int32_t H, int32_t W, int32_t blocks, int32_t site, int32_t parts, int32_t A,
                             const float* x, const float* w, const float* bias, const int32_t* action, const int32_t* parent,
                             int32_t pool_stride, float* out, int64_t* launches, int32_t* saturated, int64_t* plan);

/* Launch plan of the 256-channel tower (host only; the route MZ_TC_WIDE=3 opts 256-channel nets such as games/atari.py's
 * into): n boards of C x H x W through [a stem conv, C + 1 planes with the action plane, if stem] + `blocks` residual blocks
 * as x3 tensor-core MMAs on clusters of two CTAs, CTA r computing output channels [128 r, 128 r + 128) of `boards` boards
 * stacked in its M rows and exchanging them through distributed shared memory after every layer.  boards = 0 plans the
 * largest number of boards per CTA pair that fits, boards > 0 forces that many.  Fills plan[10] = {boards per CTA pair,
 * M-tiles per CTA, threads per CTA, dynamic shared-memory bytes per CTA, weight ring stages, layers, CTAs per SM, boards per
 * wave, launches per tower call, registers per thread assumed} and returns 1; returns 0 with the reason in
 * mz_last_error(NULL) when the tower refuses the shape (C != 256, more than 16 blocks, a board beyond the M-tile or
 * shared-memory budget). */
int mz_debug_wide256_tower_plan(int32_t n, int32_t C, int32_t H, int32_t W, int32_t blocks, int32_t stem, int32_t sm_count,
                                int32_t boards, int64_t* plan);

/* Debug / parity: mz_debug_wide_tower for 256 channels (x [n][256][H][W], w the convs [256][cin][3][3] back to back with
 * cin = 257 for the dynamics stem, bias [convs][256]) on the 256-channel tower, with `boards` as for
 * mz_debug_wide256_tower_plan; plan (or NULL) as that entry fills it.  MZ_EUNSUPPORTED when the tower refuses the shape. */
int mz_debug_wide256_tower(int device, int32_t n, int32_t H, int32_t W, int32_t blocks, int32_t site, int32_t parts, int32_t A,
                           const float* x, const float* w, const float* bias, const int32_t* action, const int32_t* parent,
                           int32_t pool_stride, int32_t boards, float* out, int64_t* launches, int32_t* saturated,
                           int64_t* plan);

/* Routes of the residual heads (route argument of mz_debug_heads_plan and mz_debug_heads, plan[0]).  The network always
 * takes MZ_HEADS_PLANNED: heads_kernel<32> (one warp per sample) when C*H*W <= 1024, heads_kernel<128> (128 threads per
 * sample) otherwise, the generic route (one plain kernel per stage) when the head weights and one sample's tile exceed
 * shared memory. */
#define MZ_HEADS_PLANNED 0
#define MZ_HEADS_WARP 1             /* heads_kernel<32> */
#define MZ_HEADS_WIDE 2             /* heads_kernel<128> */
#define MZ_HEADS_GENERIC 3          /* big_*_kernel: dense states, one range only */
/* State layouts of a heads call (layout argument): dense NCHW fp32, or the tensor-core board layout (64 channels, boards up to
 * 6 x 7) of one fp16 plane or of split fp16 planes x = x_h + x_l / 2^11 */
#define MZ_LAYOUT_DENSE 0
#define MZ_LAYOUT_F16 1
#define MZ_LAYOUT_SPLIT 2

/* Launch plan of one heads call (host only) of the samples [g0, g0 + n) at a call site (MZ_TOWER_REPRESENTATION: rescale
 * only; MZ_TOWER_DYNAMICS / MZ_TOWER_DYNAMICS_POOL: reward head + rescale; MZ_TOWER_PREDICTION: value + policy heads) of C
 * channels on an H x W board.  shapes holds one row of 3 + MZ_MAX_LAYERS int32 per head of the site: {reduced channels,
 * logits, hidden layers, hidden widths...}; the first head of a site is scalarised, so its logits are 2 S + 1.  Fills plan[5]
 * = {route (MZ_HEADS_WARP / _WIDE / _GENERIC), groups per CTA, threads per CTA, grid, dynamic shared-memory bytes; the last
 * four 0 on the generic route} and returns 1; returns 0 with the reason in mz_last_error(NULL) when the shape or the forced
 * route is refused (the generic route on a board layout or with g0 != 0, a forced group that does not fit). */
int mz_debug_heads_plan(int32_t n, int32_t g0, int32_t C, int32_t H, int32_t W, int32_t site, int32_t layout, int32_t route,
                        const int32_t* shapes, int32_t sm_count, int64_t* plan);

/* Debug / parity: the heads call of one call site of resnet_inference (models.py:530-553 rescale, conv1x1 -> flatten -> MLP
 * with ELU -> logits, models.py:645-666 support_to_scalar) on host NCHW fp32 data x [n][C][H][W], encoded into `layout`,
 * through the helper the network calls.  The heads are packed from `tensors`: "h<i>.conv.weight" [rc][C] and ".bias" [rc],
 * "h<i>.fc.<2l>.weight" [out][in] and ".bias" [out] as in the reference state_dict, shaped by `shapes` (as above).  `parts`
 * (1..4, MZ_TOWER_DYNAMICS_POOL only) runs the samples in the ranges of the partitioned replay.  Outputs (NULL: not copied
 * back), each filled with NaN bytes before the launch: logits0 / logits1 [n][logits] of the site's heads, scalar [2][n]
 * (row 0 the first head's support_to_scalar), and at the rescaling sites rescaled [n][C][H][W], pool [n][pool_stride][state]
 * (the rescaled state in slot out_slot, 0 <= out_slot < pool_stride, in the layout: C*H*W floats dense, 2048 floats of
 * fp16 or 4096 of split fp16 per board) and, on the board layouts, state [n][state] (the prediction tower's input).  plan gets
 * the plan of the launch (of the first range).  MZ_EUNSUPPORTED when a range's plan is refused. */
int mz_debug_heads(int device, int32_t n, int32_t C, int32_t H, int32_t W, int32_t site, int32_t layout, int32_t route,
                   int32_t parts, const int32_t* shapes, const MzTensor* tensors, int32_t n_tensors, const float* x,
                   int32_t pool_stride, int32_t out_slot, float* logits0, float* logits1, float* scalar, float* rescaled,
                   float* pool, float* state, int64_t* plan);

/* Routes of the fully-connected networks (route argument of mz_debug_fc_net_plan and mz_debug_fc_net): fc_inference_kernel
 * as mz_initial_inference, mz_recurrent_inference and the step-wise search's pool call run it, and the two network calls of
 * the fused search kernel (its root evaluation and one simulation's recurrent inference).  Paths (plan[0]): */
#define MZ_FC_INFER_INITIAL 0
#define MZ_FC_INFER_RECURRENT 1
#define MZ_FC_INFER_POOL 2          /* parents gathered from and the new state written to a [n][pool_stride][E] pool */
#define MZ_FC_SEARCH_ROOT 3
#define MZ_FC_SEARCH_SIM 4
#define MZ_FC_PATH_INFER 0          /* fc_inference_kernel<G> */
#define MZ_FC_PATH_FIXED 1          /* the search's unrolled network of games/cartpole.py's shape (G = 16 or 32) */
#define MZ_FC_PATH_FUSED 2          /* the search's descriptors walk, the three heads side by side (equal depth) */
#define MZ_FC_PATH_SPLIT 3          /* the search's descriptors walk, the heads one after the other */

/* Launch plan (host only) of one FC network route for n samples with G lanes per sample (4, 8, 16 or 32) on sm_count SMs with
 * smem_cap bytes of shared memory per block.  `net` gives the shape (kind, encoding, action_space, support_size, layer lists)
 * and obs_elems the observation floats.  force_split (search routes) walks the layer descriptors with the heads one after
 * the other, even for the unrolled shape or heads of equal depth; the network never does.  Fills plan[5] = {path (MZ_FC_PATH_*), G, threads per CTA, grid, dynamic shared-memory
 * bytes} and returns 1; returns 0 with the reason in mz_last_error(NULL) when the shape is refused (it does not fit in
 * shared memory, or a search route with action_space > G). */
int mz_debug_fc_net_plan(const MzNetDesc* net, int32_t obs_elems, int32_t G, int32_t route, int32_t force_split, int32_t n,
                         int32_t sm_count, int64_t smem_cap, int64_t* plan);

/* Debug / parity: one FC network route for n samples, weights packed from `tensors` named as in the reference state_dict.
 * in: observations [n][obs_elems] (MZ_FC_INFER_INITIAL, MZ_FC_SEARCH_ROOT) or parent states [n][E]; action [n] on the
 * recurrent routes; on MZ_FC_INFER_POOL parent [n] is each sample's pool slot, where the entry puts its parent state, and
 * out_slot the slot the kernel writes (pool: [n][pool_stride][E] back).  Outputs (NULL: not copied back), each filled with
 * NaN bytes before the launch: raw [n][E] the state before the rescale (search routes), hidden [n][E] after it, reward /
 * value logits [n][2S+1], policy logits [n][A] (the unrolled path keeps its logits in registers and writes none), prior
 * [n][A] (search routes), value [n] and reward [n] (the search's root has none; the initial inference writes the value
 * transform of 0).  plan gets the plan of the launch.  MZ_EUNSUPPORTED when the plan is refused. */
int mz_debug_fc_net(int device, const MzNetDesc* net, int32_t obs_elems, const MzTensor* tensors, int32_t n_tensors, int32_t G,
                    int32_t route, int32_t force_split, int32_t n, const float* in, const int32_t* action, const int32_t* parent,
                    int32_t pool_stride, int32_t out_slot, float* raw, float* hidden, float* reward_logits, float* value_logits,
                    float* policy_logits, float* prior, float* value, float* reward, float* pool, int64_t* plan);

/* Launch plan of the DownsampleCNN stem (downsample = 2, models.py:278-297; host only) for n boards of `in` planes of H x W
 * and C channels on sm_count SMs.  Fills plan[36] = {h, w (hidden board, ceil(H / 16) x ceil(W / 16)), mid (conv1's
 * channels, (in + C) / 2)}, then per stage (conv1 + pool1 at plan[3], conv2 + pool2 + average at plan[19]) {kernel, stride,
 * conv rows, conv columns, pooled rows, pooled columns, output channels per CTA, pooled rows per band, bands (grid z), boards
 * per CTA, cin chunk, conv pixels per thread, threads per CTA, grid x, grid y, dynamic shared-memory bytes}, and returns 1;
 * returns 0 with the reason, naming the failing stage, in mz_last_error(NULL) when the reference's module cannot run the
 * geometry (mz_create refuses such a net). */
int mz_debug_cnn_stem_plan(int32_t n, int32_t in, int32_t C, int32_t H, int32_t W, int32_t sm_count, int64_t* plan);

/* Debug / parity: the DownsampleCNN stem alone on host NCHW fp32 data, through the launcher of the network: x
 * [n][in][H][W]; w1 [mid][in][k][k] with k = 2 ceil(H / 16), b1 [mid], w2 [C][mid][5][5], b2 [C] as in the reference
 * state_dict (features.0 and features.3); out [n][C][ceil(H / 16)][ceil(W / 16)], filled with NaN on the device before the
 * launch.  plan (or NULL) gets the plan launched, as mz_debug_cnn_stem_plan fills it.  MZ_EUNSUPPORTED for a geometry the
 * plan refuses. */
int mz_debug_cnn_stem(int device, int32_t n, int32_t in, int32_t C, int32_t H, int32_t W, const float* x, const float* w1,
                      const float* b1, const float* w2, const float* b2, float* out, int64_t* plan);

/* Debug / parity: the DownSample stem (downsample = 1, models.py:233-275) alone on host NCHW fp32 data, through the
 * network's weight packer and launcher: x [n][in][H][W]; w the 18 convs' [cout][cin][3][3] weights one after another
 * in execution order (conv1 in -> C/2 at stride 2; resblocks1.0.conv1, .conv2, resblocks1.1.conv1, .conv2 at C/2;
 * conv2 C/2 -> C at stride 2; resblocks2.0 to .2 and resblocks3.0 to .2, conv1 then conv2 each, at C), BatchNorm
 * folded in; bias their [cout] biases in the same order, conv1's and conv2's zero (the reference's convs have none).
 * out [n][C][ceil(H / 16)][ceil(W / 16)].  stages (or NULL) gets, one after another, the outputs of conv1 and of
 * resblocks1 ([n][C/2][H1][W1] each, H1 = ceil(H / 2)), of conv2 and of resblocks2 ([n][C][H2][W2], H2 = ceil(H1 / 2)),
 * of the first pool and of resblocks3 ([n][C][H3][W3], H3 = ceil(H2 / 2)).  Every device buffer but the input starts
 * as NaN.  C must be a positive multiple of 8; MZ_EUNSUPPORTED when a conv's launch plan is refused. */
int mz_debug_downsample(int device, int32_t n, int32_t in, int32_t C, int32_t H, int32_t W, const float* x, const float* w,
                        const float* bias, float* out, float* stages);

/* Arithmetic the handle's search path computes in, e.g. "f32 nets + f64 tree statistics" (bench.py's dtype). */
const char* mz_numerics(const MzHandle* h);

/* ------------------------------------------------------------------------------------------------------------------
 * Device-resident self-play (SURVEY.md 8f-1): the per-move loop of SelfPlay.play_game (self_play.py:110-183) for
 * max_games environments whose state lives on the GPU.  One move = [batched MCTS.run on the device-side observations]
 * -> [visit-count sampling, self_play.py:222-245] -> [environment step] -> [one struct-of-arrays record per game].
 * A finished game (done, or max_moves reached, self_play.py:129-131) is packed into a pinned host staging area by the
 * kernel that detects it and its slot starts a new game with a fresh global id (old id + game_id_stride); the host reads
 * finished games only.  Root noise, the first simulation's tie and the action sample come from Philox4x32-10 streams
 * keyed (seed, game id, move), so a game's history does not depend on the batch or on the number of ranks.
 * With stacked_observations = s > 0 the search input is GameHistory.get_stacked_observations(-1, s, A)
 * (self_play.py:513-550), built on the device from the game's records: the observation of move t, then for
 * k = 1..s, p = t - k, the observation after move p and a plane filled with (float)((double)action_p / A) (C + 1 zero
 * planes when p < 0).  The handle's obs_elems must be (C * (s + 1) + s) * H * W for the environment's C planes of
 * H x W; the records and the staged blocks hold the environment's own C * H * W observation. */
enum { MZ_ENV_CARTPOLE = 0, MZ_ENV_TICTACTOE = 1, MZ_ENV_CONNECT4 = 2, MZ_ENV_GOMOKU = 3, MZ_ENV_TWENTYONE = 4,
       MZ_ENV_SIMPLE_GRID = 5 };
/* not an environment of the library: any game, stepped by the caller (mz_selfplay_begin_host) */
#define MZ_ENV_HOST 6
/* Gridworld (games/gridworld.py), a device environment numbered after MZ_ENV_HOST */
#define MZ_ENV_GRIDWORLD 7

typedef struct MzSelfPlayDesc {
    int32_t env;                  /* MZ_ENV_*: games/cartpole.py:131-174 (restated cart-pole physics),
                                     games/tictactoe.py:243-306, games/connect4.py:220-305,
                                     games/gomoku.py:220-292 (s x s, five in a row; the mover is paid reward_scale
                                     whenever the game ends, a full board included; the side is taken from the
                                     handle, s = isqrt(action_space), which must be a square with 5 <= s <= 16:
                                     the reference's board_size, 11 by default),
                                     games/twentyone.py:228-303 with Game.step's x10 (one player; cards from the Philox
                                     stream tag 0x7169E006 at counter (game id, draw k, 0, game id >> 32): card =
                                     1 + floor(12 u), value min(card, 10); draw 0 = the player's first card, 1 = the
                                     dealer's, then hits and the dealer's draws in the reference's order),
                                     games/simple_grid.py:125-229 (one player; 3x3 grid, one-hot observation of 9),
                                     MZ_ENV_GRIDWORLD: games/gridworld.py's restatement of gym_minigrid's
                                     MiniGrid-Empty-Random-6x6-v0 behind ImgObsWrapper (one player; 3 actions; the
                                     7x7x3 view [x'][y'][c] as 7 planes of 7x3; reward 1 - 0.9 * step_count / 144 in
                                     fp64 on reaching the goal, rounded to float; reward_scale unused; placement
                                     from the Philox stream tag 0x7169E007 at counter (game id, draw k, 0, game id
                                     >> 32): draw 0 gives the floor(15 u)-th free cell, x = 1 + i % 4,
                                     y = 1 + i / 4, draw 1 the direction floor(4 u)) */
    int32_t max_moves;            /* config.max_moves */
    int32_t temperature_threshold;/* config.temperature_threshold, 0 = None (self_play.py:153-156) */
    int32_t reward_scale;         /* board games: reward of the winning move (tictactoe.py:144: 20, connect4.py:144: 10,
                                     gomoku: 1); Twenty-One and Simple Grid: Game.step's factor, 10 */
    int64_t first_game_id;        /* slot g plays the global games first_game_id + g + k * game_id_stride, k = 0, 1, ... */
    int64_t game_id_stride;       /* 0 = max_games; world_size * max_games keeps ids unique across ranks */
    /* Initial prioritised-replay priorities |root_value - n-step target| ** PER_alpha of every position of a finished
     * game (ReplayBuffer.save_game + compute_target_value, replay_buffer.py:33-51,230-262), evaluated by the warp that packs
     * the game.  td_steps = 0: not computed.  discount_pow[k] = config.discount ** k for k = 0..td_steps, computed by the
     * caller (Python's own pow, so the products are the reference's); per_alpha must be 0.5 or 1 (an exact sqrt / identity). */
    int32_t td_steps;
    int32_t stacked_observations; /* config.stacked_observations, >= 0; 0 = the search sees the observation alone */
    double per_alpha;
    const double* discount_pow;
    uint64_t staging_bytes;       /* capacity of the finished-game staging area, 0 = library default (4x the bytes of
                                     every slot finishing a maximum-length game at once, within [16 MiB, 64 MiB];
                                     the library keeps two such areas) */
} MzSelfPlayDesc;

/* Optional per-move overrides (HOST pointers, n = max_games; only with n_moves == 1).  Parity tests drive the
 * environments with recorded actions and replay the host loop's draws through them. */
typedef struct MzSelfPlayInject {
    const int32_t* forced_action; /* [n] play this action instead of sampling (entries < 0: sample) */
    const double* uniform;        /* [n] the uniform of the action sample instead of the Philox draw */
    const double* noise;          /* [n, A] root Dirichlet noise by action id instead of the device draw */
    const int32_t* first_index;   /* [n] first-simulation pick instead of the device draw */
} MzSelfPlayInject;

typedef struct MzSelfPlayStats {
    int64_t env_steps;            /* moves played since mz_selfplay_begin (all slots) */
    int64_t games_finished;       /* games packed into the staging area since mz_selfplay_begin */
    int64_t staged_bytes;         /* bytes waiting in the staging area */
    int32_t staged_games;         /* games waiting in the staging area */
    int32_t parked_slots;         /* times a finished game did not fit into the staging area during the last call
                                     (it waits in its slot and is staged after the next drain) */
    double device_ms;             /* device time of the last mz_selfplay_moves call */
    int64_t staging_capacity;     /* bytes the staging area holds (callers size their moves-per-call from it) */
} MzSelfPlayStats;

/* Current device-side view of the environments (HOST output pointers, any may be NULL). */
typedef struct MzSelfPlayPeek {
    float* obs;                   /* [n, obs_elems] input the next search will see (the stacked input when
                                     stacked_observations > 0) */
    uint8_t* legal_mask;          /* [n, A] */
    int32_t* to_play;             /* [n] */
    int64_t* game_id;             /* [n] */
    int32_t* move_index;          /* [n] moves played in the slot's current game */
    int32_t* last_action;         /* [n] action played by the last move (-1 before the first) */
} MzSelfPlayPeek;

/* Staged games are self-describing blocks laid out back to back (all little endian, 8-byte aligned):
 *   int64 game_id; int32 slot; int32 length T; int32 first_to_play; int32 obs_elems O; int32 actions A; int32 bytes;
 *   double root_value[T]; int32 visit_counts[T][A]; int32 action[T]; float reward[T]; int32 to_play[T] (after the move);
 *   float priority[T] (zeros unless td_steps > 0); float observation[T+1][O] (index 0 = reset observation); padding to 8.
 * Loops begun with mz_selfplay_begin_host_window stage O = 0 and no observations: the caller kept them.
 * = the fields of GameHistory (self_play.py:479-511) minus the dummy first entries.
 * In test-mode games (mz_selfplay_begin_vs, mz_selfplay_begin_host_vs or mz_selfplay_begin_user_vs with an opponent) a move the
 * opponent played has root_value NaN and all
 * visit counts 0 (store_search_statistics(None), self_play.py:496-511: root_values holds None there and child_visits
 * has no row); its action, reward, to_play and observation are recorded like MuZero's. */
#define MZ_STAGED_HEADER_BYTES 32

/* replaces the per-move body of SelfPlay.play_game / continuous_self_play for a whole batch (self_play.py:31-183) */
int mz_selfplay_begin(MzHandle* h, const MzSelfPlayDesc* desc);

/* Opponents of test-mode games (SelfPlay.select_opponent_action, self_play.py:188-220), board games only (Gomoku: RANDOM
 * only, the reference's Gomoku has no expert_agent):
 *   EXPERT  Game.expert_agent (games/tictactoe.py:308-349, games/connect4.py:307-343): a win, else the last block the
 *           scan finds, else the random default;
 *   RANDOM  the random default: the legal action with index floor(u * n_legal) in ascending order, u from the Philox
 *           stream tag 0x7169E005 at counter (game id, move, 0, game id >> 32). */
enum { MZ_OPPONENT_SELF = 0, MZ_OPPONENT_EXPERT = 1, MZ_OPPONENT_RANDOM = 2 };

/* play_game(temperature, threshold, False, opponent, muzero_player) (self_play.py:110-183) for a whole batch:
 * mz_selfplay_begin with the opponent playing every move whose to_play is not muzero_player, in the same step, so
 * every search is at MuZero's turn (the opponent opens a game when muzero_player is 1).  max_moves counts both sides'
 * moves, and so does MzSelfPlayStats.env_steps.  mz_selfplay_begin(h, d) is mz_selfplay_begin_vs(h, d, MZ_OPPONENT_SELF, 0).
 * Refused: an opponent on a one-player game (CartPole, Twenty-One, Simple Grid, Gridworld), muzero_player outside {0, 1}, td_steps > 0
 * with an opponent, stacked_observations < 0, a handle whose action space or obs_elems does not fit the environment and
 * stacked_observations (MZ_EINVAL); an unknown opponent, EXPERT on Gomoku (MZ_EUNSUPPORTED).  The opponent's moves are
 * part of the stacked history like MuZero's. */
int mz_selfplay_begin_vs(MzHandle* h, const MzSelfPlayDesc* desc, int32_t opponent, int32_t muzero_player);
int mz_selfplay_moves(MzHandle* h, int32_t n_moves, double temperature, const MzSelfPlayInject* inject, MzSelfPlayStats* stats);
/* the same in two halves, so the host can work while the device plays: enqueue returns at once, wait synchronises */
int mz_selfplay_enqueue(MzHandle* h, int32_t n_moves, double temperature);
int mz_selfplay_wait(MzHandle* h, MzSelfPlayStats* stats);
/* pointer to the staged games (pinned host memory owned by the library) and marks them consumed.  The library keeps
 * two staging areas and swaps them here: the games returned stay intact during the NEXT mz_selfplay_moves / enqueue and
 * are overwritten by the one after the next drain.  `index` (may be NULL) receives a table of n_games pairs of uint64:
 * {byte offset of the game's block, (slot << 32) | length}, so a consumer can address any game without walking. */
int mz_selfplay_drain(MzHandle* h, const void** data, uint64_t* bytes, int32_t* n_games, const uint64_t** index);
int mz_selfplay_peek(MzHandle* h, const MzSelfPlayPeek* out);

/* Host-stepped games (env = MZ_ENV_HOST): the device loop for a game whose environment only the caller can step (any
 * game plug-in).  Search, the action sample (the same Philox stream), the per-move records, stacked observations, PER
 * priorities and the packed hand-over stay on the device; each move is
 *   mz_selfplay_host_act      one batched search and the action of every playing slot, -1 for a slot that is not
 *                             playing (its finished game is parked: the staging area was full); do not step those
 *   [the caller steps the environments of the slots with action >= 0]
 *   mz_selfplay_host_observe  the step's rows for the whole batch (rows of slots that did not play are ignored):
 *                             obs [n][C*H*W], reward [n] (the game's reward rounded once to float), done [n],
 *                             legal [n][A], to_play [n] after the move.  finished [n] receives 1 for the slots whose game
 *                             ended (done, or max_moves reached) and was packed: reset their environments
 *   mz_selfplay_host_restart  the first rows of the next game of the slots of `which` (a subset of those reported
 *                             finished); that game's id is the slot's previous id + game_id_stride
 * A game that ended but did not fit into the staging area is reported finished by a later observe, after a drain.
 * Every slot reported finished must be restarted before the next act; calls out of this order fail with MZ_ESTATE, and
 * so do mz_selfplay_moves / _enqueue on a host-stepped loop.  mz_selfplay_drain and mz_selfplay_peek work as above. */
typedef struct MzHostEnvDesc {
    int32_t obs_channels;         /* the environment's observation is obs_channels x obs_h x obs_w floats; the stack's */
    int32_t obs_h;                /* action planes are obs_h x obs_w (GameHistory.get_stacked_observations) */
    int32_t obs_w;
} MzHostEnvDesc;

/* Starts games first_game_id + g from the caller's first rows (obs [n][C*H*W], legal [n][A], to_play [n]).  Refused
 * with MZ_EINVAL: desc->env other than MZ_ENV_HOST, an observation that with stacked_observations does not give the
 * handle's obs_elems, a row without a legal action, a to_play outside the players (mz_selfplay_begin_vs refuses
 * MZ_ENV_HOST with an opponent other than MZ_OPPONENT_SELF: test-mode games of host-stepped games begin with
 * mz_selfplay_begin_host_vs).  MZ_ENOMEM, with the bytes per slot, when the records ([max_games][max_moves + 1]
 * observations) do not fit on the device. */
int mz_selfplay_begin_host(MzHandle* h, const MzSelfPlayDesc* desc, const MzHostEnvDesc* env, const float* obs,
                           const uint8_t* legal, const int32_t* to_play);
/* mz_selfplay_begin_host, but the caller keeps each game's observations: the device holds a window of the last
 * stacked_observations + 1 observations per slot, and staged blocks carry obs_elems = 0 and no observation section.
 * For image games with long episodes (games/atari.py: 27000 moves of 3 x 96 x 96 frames, 2.99 GB per slot with the whole
 * game on the device, 3.65 MB with the window of 33).  The stacked inputs, records, priorities and every other call are
 * those of mz_selfplay_begin_host, and so are its refusals; MZ_ENOMEM counts the window's observations per slot. */
int mz_selfplay_begin_host_window(MzHandle* h, const MzSelfPlayDesc* desc, const MzHostEnvDesc* env, const float* obs,
                                  const uint8_t* legal, const int32_t* to_play);
int mz_selfplay_host_act(MzHandle* h, double temperature, const MzSelfPlayInject* inject, int32_t* actions);
int mz_selfplay_host_observe(MzHandle* h, const float* obs, const float* reward, const uint8_t* done, const uint8_t* legal,
                             const int32_t* to_play, uint8_t* finished, MzSelfPlayStats* stats);
int mz_selfplay_host_restart(MzHandle* h, const uint8_t* which, const float* obs, const uint8_t* legal,
                             const int32_t* to_play);

/* Test-mode games of host-stepped games: play_game(temperature, threshold, False, opponent, muzero_player) as
 * mz_selfplay_begin_vs plays them, with the opponent's moves stepped by the caller.  window = 0 begins like
 * mz_selfplay_begin_host, 1 like mz_selfplay_begin_host_window; with MZ_OPPONENT_SELF and muzero_player 0 the call IS
 * that entry point.  Refused: those entry points' refusals and mz_selfplay_begin_vs's (an unknown opponent:
 * MZ_EUNSUPPORTED; muzero_player outside {0, 1}, td_steps > 0 with an opponent: MZ_EINVAL), an opponent on a handle of
 * one player and window outside {0, 1} (MZ_EINVAL).
 * With an opponent, every begin, observe and restart is followed by the opponent phase, repeated while moves are due:
 *   mz_selfplay_host_opponent_turn  defaults [n] receives, for every slot whose game is in play and whose to_play is not
 *                                   muzero_player, the random default of MZ_OPPONENT_RANDOM (the same Philox draw as
 *                                   the device opponent's, on the slot's published legal mask), -1 for the others.
 *                                   Returns the number of such slots; 0 ends the phase and MuZero moves next
 *   mz_selfplay_host_opponent_act   the opponent's move of every such slot: actions[g] (the caller's EXPERT, which may
 *                                   fall back to the default), or the default when actions is NULL (the RANDOM
 *                                   opponent).  played [n] receives the moves, -1 for a slot without one; the move is
 *                                   recorded with root_value NaN and zero visit counts and counts in env_steps
 *   [the caller steps the environments of the slots with played >= 0]
 *   mz_selfplay_host_observe        as above; it may finish games, reported and restarted as usual
 * max_moves counts both sides' moves.  mz_selfplay_host_act answers MZ_ESTATE until a turn returned 0, and so do the
 * opponent calls out of this order or on a loop without an opponent.  MZ_EINVAL: NULL actions with the EXPERT opponent,
 * an action that is not legal in its slot's published mask (nothing is recorded; the call can be made again). */
int mz_selfplay_begin_host_vs(MzHandle* h, const MzSelfPlayDesc* desc, const MzHostEnvDesc* env, int32_t opponent,
                              int32_t muzero_player, int32_t window, const float* obs, const uint8_t* legal,
                              const int32_t* to_play);
int mz_selfplay_host_opponent_turn(MzHandle* h, int32_t* defaults);
int mz_selfplay_host_opponent_act(MzHandle* h, const int32_t* actions, int32_t* played);

/* User environments (env = MZ_ENV_USER): the device loop for a game plug-in that brings its environment as CUDA source.
 * The library compiles the source with NVRTC (-arch=sm_90a -std=c++17 -fmad=false, the built-in environments' flags)
 * behind the prelude csrc/user_env.cuh, which states the contract: the source defines
 *   __device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row);
 *   __device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row);
 * on the slot's own state_bytes of device memory; MzEnvCtx carries the handle's seed, the slot's game id, the move index
 * and the slot, MzEnvRow the slot's observation, reward, done, legal-mask and to_play entries, and the prelude exposes
 * philox_uniform53, the Philox draw of the built-in environments.  Each move is then the host-stepped loop's with the
 * step on the device: search, the action sample and the search records (as mz_selfplay_host_act), the step kernel, the
 * rest of the records, packing and stacking (as mz_selfplay_host_observe), the reset kernel on the slots whose game was
 * packed and their next game's first rows (as mz_selfplay_host_restart); nothing crosses to the host but the counters
 * at the end of the call.  NVRTC is loaded with dlopen("libnvrtc.so.12") on first use: without it these calls fail
 * with MZ_EUNSUPPORTED and every other entry point works. */
#define MZ_ENV_USER 8
#define MZ_USER_ENV_MAX_STATE_BYTES 4096
typedef struct MzUserEnvDesc {
    const char* source;           /* NUL-terminated CUDA source defining mz_env_reset and mz_env_step */
    int32_t state_bytes;          /* bytes of environment state per slot, 0 .. MZ_USER_ENV_MAX_STATE_BYTES */
    int32_t obs_channels;         /* the observation is obs_channels x obs_h x obs_w floats (as MzHostEnvDesc) */
    int32_t obs_h;
    int32_t obs_w;
} MzUserEnvDesc;

/* Compiles env->source (or takes it from the handle's cache of sources compiled before), resets every slot (games
 * first_game_id + g) and begins the loop as mz_selfplay_begin_host does, stacked_observations and device priorities
 * included.  Refused with MZ_EINVAL: desc->env other than MZ_ENV_USER, state_bytes outside [0,
 * MZ_USER_ENV_MAX_STATE_BYTES], a source that does not compile or lacks one of the two functions (NVRTC's log in
 * mz_last_error), mz_selfplay_begin_host's refusals, and a reset that left a slot without a legal action or with a
 * to_play outside the players.  MZ_EUNSUPPORTED: no NVRTC. */
int mz_selfplay_begin_user(MzHandle* h, const MzSelfPlayDesc* desc, const MzUserEnvDesc* env);
/* mz_selfplay_moves for a loop begun with mz_selfplay_begin_user (mz_selfplay_moves refuses those; mz_selfplay_enqueue /
 * _wait, _drain and _peek serve both).  A finished game that does not fit into the staging area is parked as in the
 * device loop.  MZ_EINVAL when the environment wrote a row the loop cannot play (a game in play without a legal action,
 * a to_play outside the players): such a game was ended there, and the loop should be begun again. */
int mz_selfplay_user_moves(MzHandle* h, int32_t n_moves, double temperature, const MzSelfPlayInject* inject,
                           MzSelfPlayStats* stats);
/* Test-mode games of user environments: play_game(temperature, threshold, False, opponent, muzero_player) as
 * mz_selfplay_begin_vs plays them, with the opponent's moves stepped by the source's mz_env_step.  With MZ_OPPONENT_SELF
 * and muzero_player 0 the call IS mz_selfplay_begin_user.  EXPERT needs a source that defines the macro MZ_ENV_EXPERT
 * and (csrc/user_env_expert.cuh)
 *   __device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action);
 * the opponent's move in the slot's current position: row is the published row (observation, legal mask, to_play; not
 * to be written), ctx.move the index of the move about to be played, default_action the random default of
 * MZ_OPPONENT_RANDOM (the same Philox draw), so an expert that falls back to it falls back as the built-in experts do.
 * Each move of mz_selfplay_user_moves / _enqueue then runs on the device with no host synchronisation: the search and
 * MuZero's moves (slots whose to_play is not muzero_player do not move), then two opponent passes (the random default,
 * the expert for EXPERT, recorded with root_value NaN and zero visit counts, the user step, observe, reset and
 * restart); begin runs the two passes too, so the opponent opens the games where it moves first.  The second pass
 * opens the games the first one ended, so games whose sides alternate are played in the same moves as by
 * mz_selfplay_begin_vs.  A slot whose opponent moves a third time in a row, or whose side to move is MuZero's again
 * after MuZero moved, waits for the next pass of its side; its games do not change, since every draw is keyed by game
 * id and move.  max_moves counts both sides' moves, and so does MzSelfPlayStats.env_steps.
 * Refused: mz_selfplay_begin_user's refusals and mz_selfplay_begin_vs's (an unknown opponent: MZ_EUNSUPPORTED;
 * muzero_player outside {0, 1}, td_steps > 0 with an opponent: MZ_EINVAL), an opponent on a handle of one player
 * (MZ_EINVAL), EXPERT on a source without mz_env_expert (MZ_EUNSUPPORTED); all before the running loop is dropped.
 * An expert move out of range or not legal in the slot's mask is replaced by the default and fails the call (begin or
 * moves) with MZ_EINVAL, as a bad row does; begin the loop again. */
int mz_selfplay_begin_user_vs(MzHandle* h, const MzSelfPlayDesc* desc, const MzUserEnvDesc* env, int32_t opponent,
                              int32_t muzero_player);
/* Debug, host only (no device needed): compiles source as mz_selfplay_begin_user does.  log (may be NULL) receives
 * NVRTC's log, ptxas's resource report included, truncated to log_bytes - 1 bytes and NUL-terminated; info (may be
 * NULL) receives info[9] = {registers, stack frame bytes, spill store bytes, spill load bytes} of the reset wrapper
 * kernel, the same of the step wrapper kernel, and NVRTC's version as 1000 * major + 10 * minor (-1 for a count the log
 * does not give).  MZ_EINVAL on a compile failure or a missing function, MZ_EUNSUPPORTED without NVRTC. */
int mz_debug_user_env_compile(const char* source, char* log, int64_t log_bytes, int32_t* info);
/* Debug, host only: mz_debug_user_env_compile with info[14]: info[0..8] as there, info[9] = 1 when the expert wrapper
 * was compiled (the source defines MZ_ENV_EXPERT), info[10..13] {registers, stack frame bytes, spill store bytes,
 * spill load bytes} of it (-1 without one).  A source that defines MZ_ENV_EXPERT but not mz_env_expert: MZ_EINVAL. */
int mz_debug_user_env_expert_compile(const char* source, char* log, int64_t log_bytes, int32_t* info);
/* NVRTC compiles made for this handle's user environments so far (a begin with a cached source makes none) */
int64_t mz_debug_user_env_compiles(const MzHandle* h);

/* Debug / parity: the device opponent (MZ_OPPONENT_EXPERT or MZ_OPPONENT_RANDOM) of env (MZ_ENV_TICTACTOE,
 * MZ_ENV_CONNECT4, or MZ_ENV_GOMOKU with MZ_OPPONENT_RANDOM only, on its default 11 x 11 board: this call has no handle
 * to read another side from) on n host positions.  board is [n][H*W] of +1 / -1 / 0 (row 0 = bottom), player [n] the side to
 * move (+1 / -1).  The random default is the pick for uniform[i], or default_action[i] when default_action is not NULL
 * (one of the two must be given).  out [n] receives the actions. */
int mz_debug_opponent_action(int device, int32_t env, int32_t opponent, int32_t n, const int8_t* board,
                             const int8_t* player, const double* uniform, const int32_t* default_action, int32_t* out);

#ifdef __cplusplus
}
#endif
#endif /* MZB200_H */
