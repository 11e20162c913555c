// The environment contract of plug-in games whose environment is CUDA source (mz_selfplay_begin_user, include/mzb200.h).
//
// NVRTC compiles this header in front of every user source (--pre-include) with -arch=sm_90a -std=c++17 -fmad=false,
// the flags the built-in environments of selfplay.cu are compiled with, so a restated environment can match them bit
// for bit.  It includes nothing but philox.cuh, which NVRTC is given alongside.  The library includes it for
// MzUserEnvArgs, the argument block of the two wrapper kernels.
//
// A user source defines
//   __device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row);
//   __device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row);
// reset starts game ctx.game_id in slot ctx.slot: it fills the slot's state and the row's observation, legal mask and
// to_play.  step plays `action` (legal in the row's mask): it updates the state and writes the row after the move.
// Before reset the row's legal mask is all ones and to_play 0; before step its reward and done are 0; whatever a call
// does not write keeps those values (step: the row of the previous move).  A row that ends the game (done = 1) may have
// no legal action; a reset's row, and a step's row of a game still in play, must have one.  `state` is the slot's own
// MzUserEnvDesc.state_bytes bytes (16-byte aligned, zero before the slot's first reset, not cleared between games).
// One thread runs one slot; the slots of a batch run concurrently.
// For test-mode games against the EXPERT opponent a source also defines the macro MZ_ENV_EXPERT and
//   __device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action);
// (user_env_expert.cuh, compiled after the source): the opponent's move in the slot's position, from the published row
// (not to be written), with ctx.move the move about to be played and default_action the library's random default.
//
// Random draws: philox_uniform53(ctx.seed, ctx.game_id, k, c2, tag) is the draw of the built-in environments (CartPole's
// reset: k = 0, c2 = component, kTagReset; Twenty-One: k = draw index, c2 = 0, kTagCard; Gridworld: k = draw index,
// c2 = 0, kTagPlace).  A user environment's own draws should take a tag of its own.
#pragma once
#ifdef __CUDACC_RTC__
typedef signed char int8_t;
typedef unsigned char uint8_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
#else
#include <stdint.h>
#endif
#ifndef MZ_DEVINL
#define MZ_DEVINL __device__ __forceinline__
#endif

#include "philox.cuh"

struct MzEnvCtx {
    uint64_t seed;             // the handle's seed (MzSearchDesc.seed)
    int64_t game_id;           // the slot's global game id
    int32_t move;              // reset: 0; step: moves played in the game before this one
    int32_t slot;
};

struct MzEnvRow {
    float* obs;                // [obs_elems] the observation after the reset / the move (channels x height x width)
    float* reward;             // step: the move's reward
    uint8_t* done;             // step: 1 when the move ended the game
    uint8_t* legal;            // [actions] 1 for the actions legal in the next move
    int32_t* to_play;          // the player to move next, in [0, num_players)
    int32_t obs_elems, actions, num_players;
};

using mz::philox_uniform53;
using mz::kTagReset;
using mz::kTagCard;
using mz::kTagPlace;

// the argument block of the wrapper kernels (one per launch, by value)
struct MzUserEnvArgs {
    unsigned char* state;      // [B][state_stride]
    int64_t state_stride;
    int32_t B, O, A, P;
    uint64_t seed;
    const int64_t* game_id;    // [B] the slot's current game
    const int32_t* move;       // [B] moves played in it
    const int32_t* action;     // step: [B] the move's action, < 0 for a slot not playing it
    const uint8_t* which;      // reset: [B] the slots to reset (their next game: game_id + id_stride), or nullptr: every
                               // slot, game first_game_id + g
    int64_t first_game_id, id_stride;
    float* obs;                // [B][O] the rows the loop takes (selfplay.cu's HostRows)
    float* reward;             // [B]
    uint8_t* done;             // [B]
    uint8_t* legal;            // [B][A]
    int32_t* to_play;          // [B]
    unsigned long long* bad;   // rows the loop could not play: counted here and repaired (see mz_env_check)
};

#ifdef MZ_USER_ENV_KERNELS
__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row);
__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row);

MZ_DEVINL MzEnvRow mz_env_row(const MzUserEnvArgs& a, int g) {
    return MzEnvRow{a.obs + (int64_t)g * a.O, a.reward + g, a.done + g, a.legal + (int64_t)g * a.A, a.to_play + g,
                    a.O, a.A, a.P};
}

// A row the search cannot take (a game in play without a legal action, a to_play outside the players) is counted in
// *bad, which fails the library call, and repaired so that nothing reads out of bounds: to_play 0, and the game ends
// (step) or gets every action (reset).
MZ_DEVINL void mz_env_check(const MzUserEnvArgs& a, MzEnvRow& r, bool reset) {
    bool bad = *r.to_play < 0 || *r.to_play >= a.P;
    if (bad) *r.to_play = 0;
    if (reset || !*r.done) {
        bool any = false;
        for (int k = 0; k < a.A; ++k) any |= r.legal[k] != 0;
        if (!any) {
            bad = true;
            if (reset) for (int k = 0; k < a.A; ++k) r.legal[k] = 1;
            else *r.done = 1;
        }
    }
    if (bad) atomicAdd(a.bad, 1ull);
}

extern "C" __global__ void __launch_bounds__(128) mz_user_env_reset(const MzUserEnvArgs a) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.B || (a.which && !a.which[g])) return;
    const MzEnvCtx ctx{a.seed, a.which ? a.game_id[g] + a.id_stride : a.first_game_id + g, 0, g};
    MzEnvRow r = mz_env_row(a, g);
    for (int k = 0; k < a.A; ++k) r.legal[k] = 1;
    *r.to_play = 0;
    *r.reward = 0.0f;
    *r.done = 0;
    mz_env_reset(a.state + g * a.state_stride, ctx, r);
    mz_env_check(a, r, true);
}

extern "C" __global__ void __launch_bounds__(128) mz_user_env_step(const MzUserEnvArgs a) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.B) return;
    const int action = a.action[g];
    if (action < 0) return;
    const MzEnvCtx ctx{a.seed, a.game_id[g], a.move[g], g};
    MzEnvRow r = mz_env_row(a, g);
    *r.reward = 0.0f;
    *r.done = 0;
    mz_env_step(a.state + g * a.state_stride, action, ctx, r);
    mz_env_check(a, r, false);
}
#endif
