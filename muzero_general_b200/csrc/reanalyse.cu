// Reanalyse on the device: the fresh root value of every position of a batch of games (mz_reanalyse_values),
// support_to_scalar(initial_inference(GameHistory.get_stacked_observations(i, s, A))[0]) (replay_buffer.py:345-366), or
// the self-play search re-run at every position (mz_reanalyse_search), the MuZero paper's Reanalyze.
//
// The positions, in game order, are cut into chunks of at most max_games.  A chunk covering positions [lo, hi) of a
// game needs that game's frame rows [max(0, lo - s), hi) and the same entries of its action history; only the first
// game of a chunk can start at lo > 0, so a chunk reads at most max_games + s rows.  Per chunk:
//   stage     host frames: the chunk's rows, actions and per-position indices are packed into one of two pinned
//             buffers and uploaded on a copy stream (device frames: the indices only, the frames are read in place)
//   stack     reanalyse_stack_kernel, one CTA per position, writes the stacked inputs into the representation's input
//             workspace (the search's input arena, max_games x obs_elems floats)
//   network   values: mz_initial_inference's network (route choice, range guard) with the value as its only output
//   search    search: reanalyse_search_inputs_kernel writes each position's legal row, to_play, game id and move index
//             next to the stacked inputs in the input arena, then mz_search's search (mz_dispatch_search, range guard)
//             runs on them; host results come back through the pinned output arena while the next chunk searches
// The next chunk is staged while the current chunk's network runs; events order the copies against the kernels that
// read the same buffer.  Peak device memory is fixed by max_games, s, O (and A): the two staging buffers.
#include <string.h>

#include <algorithm>
#include <vector>

#include "handle.h"
#include "common.cuh"
#include "stack.cuh"

namespace mz {

struct ReanalyseStackArgs {
    const float* frames;        // rows of O floats
    const int32_t* actions;     // action histories
    const int64_t* frame_row;   // [n] row of position q's own frame in frames
    const int64_t* action_at;   // [n] index of its game's action_history[i] in actions
    const int32_t* index;       // [n] i, the position's index in its game
    float* out;                 // [n][O_in]
    int O, plane, stack, A;
    int64_t O_in;
};

// One CTA per position, its threads strided over the position's O_in floats (games/atari.py: 1.26 M per position).
// The action plane is __double2float_rn(__ddiv_rn(a, A)), as in stack_fill.  The host evaluates the plane in the frame's
// dtype: float32 frames give the correctly rounded fp32 quotient, int or float64 frames the fp64 quotient, rounded to
// fp32 by .float().  For integers a and A below 2^24 both are the same float32: rounding to 53 bits and then to 24 is
// innocuous because 53 >= 2 * 24 + 2.
__global__ void reanalyse_stack_kernel(const ReanalyseStackArgs a) {
    const int q = blockIdx.x;
    const int t = a.index[q];
    const float* own = a.frames + a.frame_row[q] * a.O;
    const int64_t act0 = a.action_at[q] - t;          // index of the game's action_history[0] (may be before the window)
    float* dst = a.out + (size_t)q * a.O_in;
    for (int j = threadIdx.x; j < a.O; j += blockDim.x) dst[j] = own[j];
    const auto frame = [&](int p) { return own - (int64_t)(t - p) * a.O; };
    const auto action = [&](int p) { return a.actions[act0 + p + 1]; };
    const int tail = a.stack * (a.O + a.plane);
    for (int e = threadIdx.x; e < tail; e += blockDim.x)
        dst[a.O + e] = stack_tail_element(e, t, a.O, a.plane, a.A, frame, action);
}

struct ReanalyseSearchArgs {
    const uint8_t* legal;       // [n][A] the chunk's legal rows, or null = all legal
    const int32_t* to_play;     // [n] or null = 0
    const int64_t* game_id;     // [n] the game id of each position's game
    const int32_t* index;       // [n] i, the move index
    uint8_t* legal_out;
    int32_t *to_play_out, *move_out;
    int64_t* game_id_out;
    int n, A;
};

// The per-position search inputs of one chunk, in the search's input arena: threads strided over the n x A legal entries,
// the first n of them also write the position's to_play, game id and move index.
__global__ void reanalyse_search_inputs_kernel(const ReanalyseSearchArgs a) {
    const int total = a.n * a.A;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
        a.legal_out[k] = a.legal ? a.legal[k] : (uint8_t)1;
        if (k < a.n) {
            a.to_play_out[k] = a.to_play ? a.to_play[k] : 0;
            a.game_id_out[k] = a.game_id[k];
            a.move_out[k] = a.index[k];
        }
    }
}

}  // namespace mz

struct MzReanalyse {
    cudaStream_t copy = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr};      // upload of buffer b done (copy stream)
    cudaEvent_t consumed[2] = {nullptr, nullptr};    // stack kernel reading buffer b done (library stream)
    cudaEvent_t results = nullptr;                   // mz_reanalyse_search: a chunk's results are in the pinned arena
    unsigned char* host[2] = {nullptr, nullptr};     // pinned
    unsigned char* dev[2] = {nullptr, nullptr};
    size_t cap = 0;                                  // bytes of each buffer
};

static void free_buffers(MzReanalyse* r) {
    for (int b = 0; b < 2; ++b) {
        if (r->host[b]) cudaFreeHost(r->host[b]);
        if (r->dev[b]) cudaFree(r->dev[b]);
        r->host[b] = r->dev[b] = nullptr;
    }
    r->cap = 0;
}

void mz_reanalyse_destroy(MzHandle* h) {
    MzReanalyse* r = h->ra;
    if (!r) return;
    if (r->copy) cudaStreamSynchronize(r->copy);
    free_buffers(r);
    for (int b = 0; b < 2; ++b) {
        if (r->copied[b]) cudaEventDestroy(r->copied[b]);
        if (r->consumed[b]) cudaEventDestroy(r->consumed[b]);
    }
    if (r->results) cudaEventDestroy(r->results);
    if (r->copy) cudaStreamDestroy(r->copy);
    delete r;
    h->ra = nullptr;
}

namespace {

struct Plan {
    int n_games = 0, s = 0, O = 0, B = 0, A = 0;
    bool host = true;
    bool search = false;                            // mz_reanalyse_search: game ids, legal rows and to_play per position
    std::vector<int64_t> fo, ao, T, first;          // offsets, positions, first flat position of each game
    std::vector<int64_t> gid;                       // search: game id of each game
    int64_t total = 0;
    int64_t chunks() const { return (total + B - 1) / B; }
};

// Byte layout of one staging buffer: B positions, max_games + s frame rows of O floats with host frames (none with device
// frames, read in place), and for a search each position's game id, plus its to_play and legal row with host memory.
struct StageLayout {
    size_t frame_row, action_at, index, game_id, to_play, legal, actions, frames, bytes;
    explicit StageLayout(const Plan& P) {
        auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
        const size_t B = P.B, rows = P.host ? (size_t)P.B + P.s : 0;
        const size_t ids = P.search ? B : 0, rows_in = P.search && P.host ? B : 0;
        frame_row = 0;
        action_at = up(frame_row + B * 8);
        index = up(action_at + B * 8);
        game_id = up(index + B * 4);
        to_play = up(game_id + ids * 8);
        legal = up(to_play + rows_in * 4);
        actions = up(legal + rows_in * P.A);
        frames = up(actions + rows * 4);
        bytes = up(frames + rows * P.O * 4);
    }
};

int validate(MzHandle* h, const MzReanalyseIO* io, const char* who, bool need_values, Plan* P) {
    const std::string w(who);
    if (!h || !io) return fail(h, MZ_EINVAL, w + ": null argument");
    if (!h->weights_loaded) return fail(h, MZ_ESTATE, w + ": weights not loaded");
    if (io->mem != MZ_MEM_HOST && io->mem != MZ_MEM_DEVICE) return fail(h, MZ_EINVAL, w + ": mem must be MZ_MEM_HOST or MZ_MEM_DEVICE");
    const int n = io->n_games;
    if (n < 0) return fail(h, MZ_EINVAL, w + ": n_games < 0");
    const int64_t plane = (int64_t)h->net.obs_h * h->net.obs_w, O = io->frame_elems, s = io->stacked_observations;
    if (O < 1) return fail(h, MZ_EINVAL, w + ": frame_elems must be >= 1, got " + std::to_string(O));
    if (s < 0) return fail(h, MZ_EINVAL, w + ": stacked_observations must be >= 0, got " + std::to_string(s));
    if (O + s * (O + plane) != h->obs_elems) {
        const int64_t rest = h->obs_elems - O;
        const std::string implied = rest >= 0 && rest % (O + plane) == 0
            ? "s = " + std::to_string(rest / (O + plane))
            : std::string("no integer s (obs_elems - O is not a multiple of O + plane)");
        return fail(h, MZ_EINVAL, w + ": frames of O = " + std::to_string(O) + " floats with stacked_observations = " +
                    std::to_string(s) + " make inputs of " + std::to_string(O + s * (O + plane)) + " floats, the handle's " +
                    "networks take obs_elems = " + std::to_string(h->obs_elems) + " (plane = " + std::to_string(plane) +
                    "): for this O the handle implies " + implied);
    }
    if (n > 0 && (!io->frame_offsets || !io->action_offsets || !io->positions))
        return fail(h, MZ_EINVAL, w + ": frame_offsets, action_offsets and positions are required");
    P->n_games = n; P->s = (int)s; P->O = (int)O; P->B = h->search.max_games; P->A = h->net.action_space;
    P->host = io->mem == MZ_MEM_HOST;
    P->fo.assign(io->frame_offsets, io->frame_offsets + (n > 0 ? n + 1 : 0));
    P->ao.assign(io->action_offsets, io->action_offsets + (n > 0 ? n + 1 : 0));
    P->T.assign(io->positions, io->positions + n);
    P->first.resize(n);
    P->total = 0;
    for (int g = 0; g <= n && n > 0; ++g) {
        if (P->fo[g] < 0 || P->ao[g] < 0)
            return fail(h, MZ_EINVAL, w + ": offsets must be >= 0 (game " + std::to_string(g) + ")");
        if (g == n) break;
        if (P->fo[g + 1] < P->fo[g] || P->ao[g + 1] < P->ao[g])
            return fail(h, MZ_EINVAL, w + ": offsets must be non-decreasing: game " + std::to_string(g) + " has frame rows [" +
                        std::to_string(P->fo[g]) + ", " + std::to_string(P->fo[g + 1]) + ") and actions [" +
                        std::to_string(P->ao[g]) + ", " + std::to_string(P->ao[g + 1]) + ")");
        const int64_t T = P->T[g], F = P->fo[g + 1] - P->fo[g], Na = P->ao[g + 1] - P->ao[g];
        if (T < 0 || T > F)
            return fail(h, MZ_EINVAL, w + ": game " + std::to_string(g) + " has " + std::to_string(T) + " positions and " +
                        std::to_string(F) + " frames: positions must be in [0, frames]");
        if (T > Na)
            return fail(h, MZ_EINVAL, w + ": game " + std::to_string(g) + " has " + std::to_string(T) +
                        " positions but an action history of " + std::to_string(Na) + " (its leading 0 included)");
        P->first[g] = P->total;
        P->total += T;
    }
    if (P->total > 0 && (!io->frames || !io->actions || (need_values && !io->values)))
        return fail(h, MZ_EINVAL, w + ": frames, actions and values are required");
    // every action of the histories, leading 0 included, must be an action id
    const int64_t n_act = n > 0 ? P->ao[n] - P->ao[0] : 0;
    if (P->total > 0 && n_act > 0) {
        std::vector<int32_t> dev_copy;
        const int32_t* acts = io->actions + P->ao[0];
        if (!P->host) {
            dev_copy.resize(n_act);
            MZ_CUDA(h, cudaMemcpy(dev_copy.data(), acts, n_act * 4, cudaMemcpyDeviceToHost));
            acts = dev_copy.data();
        }
        const int A = h->net.action_space;
        for (int64_t k = 0; k < n_act; ++k)
            if (acts[k] < 0 || acts[k] >= A) {
                const int64_t at = P->ao[0] + k;
                const int g = (int)(std::upper_bound(P->ao.begin(), P->ao.end(), at) - P->ao.begin()) - 1;
                return fail(h, MZ_EINVAL, w + ": action " + std::to_string(acts[k]) + " at index " + std::to_string(at) +
                            " (game " + std::to_string(g) + ") is outside [0, " + std::to_string(A) + ")");
            }
    }
    return MZ_OK;
}

// The checks mz_reanalyse_search adds to validate's: a search handle, an output, every position with a legal action and
// a side to move of the game's players.  The game ids are taken into P.
int validate_search(MzHandle* h, const MzReanalyseSearchIO* io, Plan* P) {
    const std::string w = "mz_reanalyse_search";
    if (h->search.num_simulations < 1)
        return fail(h, MZ_ESTATE, w + ": the handle was created with num_simulations = 0 (an inference-only handle)");
    P->search = true;
    P->gid.resize(P->n_games);
    for (int g = 0; g < P->n_games; ++g) P->gid[g] = io->game_id ? io->game_id[g] : g;
    if (P->total == 0) return MZ_OK;
    if (!io->visit_counts) return fail(h, MZ_EINVAL, w + ": visit_counts is required");
    auto game_of = [&](int64_t q) {
        return (int)(std::upper_bound(P->first.begin(), P->first.end(), q) - P->first.begin()) - 1;
    };
    auto where = [&](int64_t q) {
        const int g = game_of(q);
        return "position " + std::to_string(q - P->first[g]) + " of game " + std::to_string(g) + " (flat " +
               std::to_string(q) + ")";
    };
    const int A = P->A;
    if (io->legal_mask) {
        std::vector<uint8_t> dev_copy;
        const uint8_t* m = io->legal_mask;
        if (!P->host) {
            dev_copy.resize((size_t)P->total * A);
            MZ_CUDA(h, cudaMemcpy(dev_copy.data(), m, dev_copy.size(), cudaMemcpyDeviceToHost));
            m = dev_copy.data();
        }
        for (int64_t q = 0; q < P->total; ++q)
            if (std::none_of(m + q * A, m + (q + 1) * A, [](uint8_t v) { return v != 0; }))
                return fail(h, MZ_EINVAL, w + ": " + where(q) + " has no legal action");
    }
    if (io->to_play) {
        std::vector<int32_t> dev_copy;
        const int32_t* t = io->to_play;
        if (!P->host) {
            dev_copy.resize(P->total);
            MZ_CUDA(h, cudaMemcpy(dev_copy.data(), t, (size_t)P->total * 4, cudaMemcpyDeviceToHost));
            t = dev_copy.data();
        }
        const int players = h->search.num_players;
        for (int64_t q = 0; q < P->total; ++q)
            if (t[q] < 0 || t[q] >= players)
                return fail(h, MZ_EINVAL, w + ": " + where(q) + " has to_play " + std::to_string(t[q]) + ", outside [0, " +
                            std::to_string(players) + ")");
    }
    return MZ_OK;
}

int ensure_staging(MzHandle* h, const Plan& P, const char* who) {
    MzReanalyse*& r = h->ra;
    if (!r) {
        r = new MzReanalyse();
        MZ_CUDA(h, cudaStreamCreateWithFlags(&r->copy, cudaStreamNonBlocking));
        for (int b = 0; b < 2; ++b) {
            MZ_CUDA(h, cudaEventCreateWithFlags(&r->copied[b], cudaEventDisableTiming));
            MZ_CUDA(h, cudaEventCreateWithFlags(&r->consumed[b], cudaEventDisableTiming));
        }
        MZ_CUDA(h, cudaEventCreateWithFlags(&r->results, cudaEventDisableTiming));
    }
    const StageLayout L(P);
    if (r->cap >= L.bytes) return MZ_OK;
    MZ_CUDA(h, cudaStreamSynchronize(r->copy));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    free_buffers(r);
    for (int b = 0; b < 2; ++b) {
        if (cudaMallocHost(&r->host[b], L.bytes) != cudaSuccess || cudaMalloc(&r->dev[b], L.bytes) != cudaSuccess) {
            cudaGetLastError();
            free_buffers(r);
            return fail(h, MZ_ENOMEM, std::string(who) + ": no room for two staging buffers of " + std::to_string(L.bytes) +
                        " bytes");
        }
    }
    r->cap = L.bytes;
    return MZ_OK;
}

// Packs chunk c into staging buffer b and uploads it on the copy stream; returns the chunk's positions in *n, the stack
// kernel's arguments in *a and, for a search, the inputs kernel's in *sa.
int stage(MzHandle* h, const MzReanalyseIO* io, const MzReanalyseSearchIO* sio, const Plan& P, int64_t c, int b, int* n,
          ReanalyseStackArgs* a, ReanalyseSearchArgs* sa) {
    MzReanalyse* r = h->ra;
    const StageLayout L(P);
    // the upload of chunk c - 2 from this buffer has finished before the host overwrites it
    MZ_CUDA(h, cudaEventSynchronize(r->copied[b]));
    unsigned char* hb = r->host[b];
    int64_t* frame_row = reinterpret_cast<int64_t*>(hb + L.frame_row);
    int64_t* action_at = reinterpret_cast<int64_t*>(hb + L.action_at);
    int32_t* index = reinterpret_cast<int32_t*>(hb + L.index);
    int64_t* game_id = reinterpret_cast<int64_t*>(hb + L.game_id);
    int32_t* actions = reinterpret_cast<int32_t*>(hb + L.actions);
    float* frames = reinterpret_cast<float*>(hb + L.frames);
    const int64_t lo_flat = c * P.B, hi_flat = std::min(P.total, lo_flat + P.B);
    int g = (int)(std::upper_bound(P.first.begin(), P.first.end(), lo_flat) - P.first.begin()) - 1;
    int q = 0;
    int64_t rows = 0;
    for (int64_t f = lo_flat; f < hi_flat; ++g) {
        if (P.T[g] == 0 || f >= P.first[g] + P.T[g]) continue;
        const int64_t lo = f - P.first[g], hi = std::min(P.T[g], lo + (hi_flat - f));
        const int64_t r0 = std::max<int64_t>(0, lo - P.s);
        if (P.host) {
            memcpy(frames + rows * P.O, io->frames + (P.fo[g] + r0) * P.O, (size_t)(hi - r0) * P.O * 4);
            memcpy(actions + rows, io->actions + P.ao[g] + r0, (size_t)(hi - r0) * 4);
        }
        for (int64_t i = lo; i < hi; ++i, ++q) {
            frame_row[q] = P.host ? rows + (i - r0) : P.fo[g] + i;
            action_at[q] = P.host ? rows + (i - r0) : P.ao[g] + i;
            index[q] = (int32_t)i;
            if (P.search) game_id[q] = P.gid[g];
        }
        rows += hi - r0;
        f += hi - lo;
    }
    *n = q;
    // a chunk's positions are consecutive in game order: its legal rows and to_play are one contiguous range
    const bool host_rows = P.search && P.host;
    if (host_rows && sio->legal_mask) memcpy(hb + L.legal, sio->legal_mask + lo_flat * P.A, (size_t)q * P.A);
    if (host_rows && sio->to_play) memcpy(hb + L.to_play, sio->to_play + lo_flat, (size_t)q * 4);
    const size_t bytes = P.host ? L.frames + (size_t)rows * P.O * 4 : L.actions;
    // the kernels of chunk c - 2 have read the device buffer before the upload overwrites it
    MZ_CUDA(h, cudaStreamWaitEvent(r->copy, r->consumed[b], 0));
    MZ_CUDA(h, cudaMemcpyAsync(r->dev[b], hb, bytes, cudaMemcpyHostToDevice, r->copy));
    MZ_CUDA(h, cudaEventRecord(r->copied[b], r->copy));
    unsigned char* db = r->dev[b];
    a->frames = P.host ? reinterpret_cast<const float*>(db + L.frames) : io->frames;
    a->actions = P.host ? reinterpret_cast<const int32_t*>(db + L.actions) : io->actions;
    a->frame_row = reinterpret_cast<const int64_t*>(db + L.frame_row);
    a->action_at = reinterpret_cast<const int64_t*>(db + L.action_at);
    a->index = reinterpret_cast<const int32_t*>(db + L.index);
    if (P.search) {
        sa->n = q;
        sa->index = a->index;
        sa->game_id = reinterpret_cast<const int64_t*>(db + L.game_id);
        sa->legal = !sio->legal_mask ? nullptr : P.host ? db + L.legal : sio->legal_mask + lo_flat * P.A;
        sa->to_play = !sio->to_play ? nullptr : P.host ? reinterpret_cast<const int32_t*>(db + L.to_play)
                                                       : sio->to_play + lo_flat;
    }
    return MZ_OK;
}

// The search's per-position inputs and outputs in the handle's arenas, at offsets fixed by max_games, so that every full
// chunk hands mz_dispatch_search the same pointers (one captured graph of the step-wise pipeline serves them all).
struct SearchArena {
    float* obs;                  // the stack kernel's workspace
    uint8_t* legal;
    int32_t *to_play, *move;
    int64_t* game_id;
    int32_t* visits;             // host memory: the results, copied to h_out
    double* root;
    size_t root_off;
    SearchArena(MzHandle* h, const Plan& P) {
        auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
        const size_t B = P.B;
        size_t o = up(B * h->obs_elems * 4);
        obs = reinterpret_cast<float*>(h->d_in);
        legal = h->d_in + o;                             o = up(o + B * P.A);
        to_play = reinterpret_cast<int32_t*>(h->d_in + o); o = up(o + B * 4);
        game_id = reinterpret_cast<int64_t*>(h->d_in + o); o = up(o + B * 8);
        move = reinterpret_cast<int32_t*>(h->d_in + o);
        visits = reinterpret_cast<int32_t*>(h->d_out);
        root_off = up(B * P.A * 4);
        root = reinterpret_cast<double*>(h->d_out + root_off);
    }
};

// The chunk loop of mz_reanalyse_values (sio null) and mz_reanalyse_search; debug_chunk >= 0 stops after that chunk's
// stack kernel and copies its inputs to debug_out instead of running the networks.
int reanalyse(MzHandle* h, const MzReanalyseIO* io, const MzReanalyseSearchIO* sio, int32_t debug_chunk, float* debug_out) {
    const char* who = sio ? "mz_reanalyse_search" : debug_chunk >= 0 ? "mz_debug_reanalyse_stack" : "mz_reanalyse_values";
    Plan P;
    int rc;
    if (h) MZ_CUDA(h, cudaSetDevice(h->device));
    if (sio && !io) return fail(h, MZ_EINVAL, std::string(who) + ": games is null");
    if ((rc = validate(h, io, who, debug_chunk < 0 && !sio, &P))) return rc;
    if (sio && (rc = validate_search(h, sio, &P))) return rc;
    const int64_t C = P.chunks();
    if (debug_chunk >= 0 && (debug_chunk >= C || !debug_out))
        return fail(h, MZ_EINVAL, std::string(who) + ": chunk " + std::to_string(debug_chunk) + " of a call with " +
                    std::to_string(C) + " chunks, or out is null");
    if (C == 0) return MZ_OK;
    if ((rc = ensure_staging(h, P, who))) return rc;
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    MzReanalyse* r = h->ra;
    const SearchArena S(h, P);
    float* workspace = S.obs;                                      // max_games x obs_elems floats
    float* d_values = reinterpret_cast<float*>(h->d_out);          // max_games floats (host values)
    ReanalyseStackArgs a[2];
    ReanalyseSearchArgs sa[2];
    int n[2];
    for (int b = 0; b < 2; ++b) {
        a[b].out = workspace; a[b].O = P.O; a[b].plane = h->net.obs_h * h->net.obs_w; a[b].stack = P.s;
        a[b].A = h->net.action_space; a[b].O_in = h->obs_elems;
        sa[b] = ReanalyseSearchArgs{};
        sa[b].A = P.A; sa[b].legal_out = S.legal; sa[b].to_play_out = S.to_play; sa[b].game_id_out = S.game_id;
        sa[b].move_out = S.move;
    }
    // search with host memory: chunk c's results wait in h_out until the host has queued chunk c + 1's search
    int64_t pending = -1;
    int pending_n = 0;
    auto drain = [&]() -> int {
        if (pending < 0) return MZ_OK;
        MZ_CUDA(h, cudaEventSynchronize(r->results));
        memcpy(sio->visit_counts + pending * P.B * P.A, h->h_out, (size_t)pending_n * P.A * 4);
        if (sio->root_value) memcpy(sio->root_value + pending * P.B, h->h_out + S.root_off, (size_t)pending_n * 8);
        pending = -1;
        return MZ_OK;
    };
    if ((rc = stage(h, io, sio, P, 0, 0, &n[0], &a[0], &sa[0]))) return rc;
    for (int64_t c = 0; c < C; ++c) {
        const int b = (int)(c & 1);
        MZ_CUDA(h, cudaStreamWaitEvent(h->stream, r->copied[b], 0));
        reanalyse_stack_kernel<<<n[b], 256, 0, h->stream>>>(a[b]);
        MZ_CUDA(h, cudaGetLastError());
        h->launches += 1;
        if (P.search) {
            const int blocks = std::max(1, std::min((n[b] * P.A + 255) / 256, 4 * h->sm_count));
            reanalyse_search_inputs_kernel<<<blocks, 256, 0, h->stream>>>(sa[b]);
            MZ_CUDA(h, cudaGetLastError());
            h->launches += 1;
        }
        MZ_CUDA(h, cudaEventRecord(r->consumed[b], h->stream));
        if (c == debug_chunk) {
            MZ_CUDA(h, cudaMemcpyAsync(debug_out, workspace, (size_t)n[b] * h->obs_elems * 4, cudaMemcpyDeviceToHost, h->stream));
            MZ_CUDA(h, cudaStreamSynchronize(h->stream));
            MZ_CUDA(h, cudaStreamSynchronize(r->copy));
            return MZ_OK;
        }
        if (P.search) {
            SearchCall call{};
            call.n = n[b]; call.obs = workspace; call.legal_mask = S.legal; call.to_play = S.to_play;
            call.add_noise = sio->add_exploration_noise ? 1 : 0; call.game_id = S.game_id; call.move_index = S.move;
            call.visit_counts = P.host ? S.visits : sio->visit_counts + c * P.B * P.A;
            call.root_value = !sio->root_value ? nullptr : P.host ? S.root : sio->root_value + c * P.B;
            if ((rc = mz_dispatch_search(h, call, false, false, 0))) return rc;
            // the host packs the next chunk and hands over the previous chunk's results while this one searches
            if (c + 1 < C && (rc = stage(h, io, sio, P, c + 1, b ^ 1, &n[b ^ 1], &a[b ^ 1], &sa[b ^ 1]))) return rc;
            if ((rc = drain())) return rc;
            MZ_CUDA(h, cudaStreamSynchronize(h->stream));
            if (h->res && resnet_take_saturations(h->res, h->stream) > 0) {
                // the x3 range guard, as mz_search: redo the chunk on the fp32 towers (its inputs are still in the arena)
                mz_switch_to_strict(h);
                if ((rc = mz_dispatch_search(h, call, false, false, 0))) return rc;
                MZ_CUDA(h, cudaStreamSynchronize(h->stream));
            }
            if (P.host) {
                MZ_CUDA(h, cudaMemcpyAsync(h->h_out, S.visits, (size_t)n[b] * P.A * 4, cudaMemcpyDeviceToHost, h->stream));
                if (sio->root_value)
                    MZ_CUDA(h, cudaMemcpyAsync(h->h_out + S.root_off, S.root, (size_t)n[b] * 8, cudaMemcpyDeviceToHost, h->stream));
                MZ_CUDA(h, cudaEventRecord(r->results, h->stream));
                pending = c;
                pending_n = n[b];
            }
            continue;
        }
        InferCall ic{};
        ic.n = n[b]; ic.recurrent = 0; ic.in = workspace;
        ic.value = P.host ? d_values : io->values + c * P.B;
        if (debug_chunk < 0 && (rc = mz_network_enqueue(h, ic))) return rc;
        // the host packs the next chunk while this one's network runs
        if (c + 1 < C && (rc = stage(h, io, sio, P, c + 1, b ^ 1, &n[b ^ 1], &a[b ^ 1], &sa[b ^ 1]))) return rc;
        if (debug_chunk < 0) {
            if ((rc = mz_network_guard(h, ic))) return rc;
            if (P.host) {
                MZ_CUDA(h, cudaMemcpyAsync(h->h_out, d_values, (size_t)n[b] * 4, cudaMemcpyDeviceToHost, h->stream));
                MZ_CUDA(h, cudaStreamSynchronize(h->stream));
                memcpy(io->values + c * P.B, h->h_out, (size_t)n[b] * 4);
            }
        }
    }
    if ((rc = drain())) return rc;
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    return MZ_OK;
}

}  // namespace

extern "C" int mz_reanalyse_values(MzHandle* h, const MzReanalyseIO* io) { return reanalyse(h, io, nullptr, -1, nullptr); }

extern "C" int mz_debug_reanalyse_stack(MzHandle* h, const MzReanalyseIO* io, int32_t chunk, float* out) {
    if (chunk < 0) return fail(h, MZ_EINVAL, "mz_debug_reanalyse_stack: chunk < 0");
    return reanalyse(h, io, nullptr, chunk, out);
}

extern "C" int mz_reanalyse_search(MzHandle* h, const MzReanalyseSearchIO* io) {
    if (!h || !io) return fail(h, MZ_EINVAL, "mz_reanalyse_search: null argument");
    return reanalyse(h, io->games, io, -1, nullptr);
}
