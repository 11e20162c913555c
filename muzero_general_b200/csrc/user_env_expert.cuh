// The epilogue of user environments: NVRTC compiles it after the user source (user_env.cu appends one line including
// it), so the expert wrapper sees whether the source defined MZ_ENV_EXPERT.  A source without the macro gets nothing
// from it, and its reset and step wrappers are those of the prelude alone.
//
// A source that defines MZ_ENV_EXPERT also defines
//   __device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action);
// the opponent's move of test-mode games (mz_selfplay_begin_user_vs with MZ_OPPONENT_EXPERT) in the slot's current
// position.  `row` is the published row (observation, legal mask, to_play; the function must not write it), ctx.move
// the index of the move about to be played, and default_action the library's random default (MZ_OPPONENT_RANDOM's
// draw), so an expert that falls back to it falls back as the built-in experts do.
#pragma once
#if defined(MZ_USER_ENV_KERNELS) && defined(MZ_ENV_EXPERT)
__device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action);

// One thread per slot: actions[g] = the expert's move of every slot with defaults[g] >= 0 (its opponent move is due).
// A move out of range or not legal in the slot's mask is counted in *bad, which fails the library call, and replaced by
// the default, so nothing reads out of bounds.
extern "C" __global__ void __launch_bounds__(128) mz_user_env_expert(const MzUserEnvArgs a, const int32_t* defaults,
                                                                     int32_t* actions) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.B) return;
    const int d = defaults[g];
    if (d < 0) return;
    const MzEnvCtx ctx{a.seed, a.game_id[g], a.move[g], g};
    const MzEnvRow r = mz_env_row(a, g);
    int action = mz_env_expert(a.state + g * a.state_stride, ctx, r, d);
    if (action < 0 || action >= a.A || !r.legal[action]) {
        atomicAdd(a.bad, 1ull);
        action = d;
    }
    actions[g] = action;
}
#endif
