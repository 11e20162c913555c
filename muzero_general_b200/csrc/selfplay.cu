// Device-resident self-play: the per-move loop of SelfPlay.play_game (self_play.py:110-183) for a whole batch.
//
//   move t:   [batched MCTS.run on the device-side observations]            mz_dispatch_search (fc_search.cu / pipeline.cu)
//             [select_action (self_play.py:222-245) + Game.step + record]   selfplay_step_kernel, lane 0 of the slot's warp
//             [finished games -> pinned host staging, slot restarts]        the same kernel, the whole warp
//
// Environments restated for the device (rules and observation planes of the reference):
//   CartPole   games/cartpole.py:131-174 wraps gym's CartPole-v1 (not vendored): Euler-integrated cart-pole, 20 ms step,
//              +1 reward per step, done at |x| > 2.4, |theta| > 12 deg or 500 steps; observation (1,1,4) fp32
//   TicTacToe  games/tictactoe.py:243-306; Connect4  games/connect4.py:220-305: planes [own stones of player +1,
//              stones of player -1, side to move (+1/-1)], player +1 = to_play 0 moves first, reward_scale for the mover
//              on completing a line, done on a line or a full board; Connect4 actions are columns (gravity)
//   Gomoku     games/gomoku.py:220-292: the same planes on s x s (5 <= s <= 16, s * s = |A|: the reference's
//              board_size, 11 by default), five in a row; the mover is paid reward_scale whenever the game ends, a full
//              board without a line included
//   TwentyOne  games/twentyone.py:228-303: hit (0) / stand (1); planes [player's hand, dealer's hand, 0] of 3x3; done on
//              a bust, a stand or exactly 21, then the dealer draws while at 16 or less unless the player went bust;
//              reward_scale * get_reward (Game.step's x10)
//   SimpleGrid games/simple_grid.py:125-229: 3x3 grid from (0, 0), action 0 = row + 1, 1 = column + 1, a move off the
//              edge changes nothing; one-hot observation of 9; reward_scale and done on reaching (2, 2)
//   Gridworld  games/gridworld.py's restatement of gym_minigrid's MiniGrid-Empty-Random-6x6-v0 + ImgObsWrapper (the
//              rules are written down there): 6x6 room, goal (4, 4), turn left / turn right / forward; reward
//              1 - 0.9 * step_count / 144 on reaching the goal, done there or at 144 steps; 7x7x3 egocentric view
// State per slot lives in HBM (a few dozen bytes); per-move records go to per-slot struct-of-arrays buffers
// [B][max_moves] and leave the device only when the game ends, as one packed block written by a warp straight into
// mapped pinned host memory (no per-move D2H, no host-side bookkeeping per move).
//
// Random draws: Philox4x32-10 keyed by (seed, global game id, move): root noise and first-simulation ties inside the
// search (tree.cuh), the action sample here (tag kTagAction), CartPole's reset state (tag kTagReset), the opponent's
// random default move in test-mode games (tag kTagOpponent), Twenty-One's cards (tag kTagCard, counter (game, draw k)),
// Gridworld's placement (tag kTagPlace, counter (game, draw k)).
//
// Test-mode games (mz_selfplay_begin_vs, the reference's play_game(0, ..., opponent, muzero_player),
// self_play.py:110-183): the opponent's move is played by the thread that played MuZero's, right after it (or by
// start_game when the opponent moves first), so every search runs at MuZero's turn.
//
// Stacked observations (config.stacked_observations = s > 0): the search input of a slot is [B][O_in] with
// O_in = O + s * (O + plane), the current observation (O floats) followed by the tail that stack_fill builds from the
// slot's records.  Records, staged blocks and rec_obs keep the environment's own O.
//
// Host-stepped environments (MZ_ENV_HOST, mz_selfplay_begin_host): any game plug-in, its step left to the host.  A move
// is two device halves with the host's step between them:
//   act       [batched MCTS.run] -> host_act_kernel: the action sample and the search records of move t (choose_action +
//             record_search, slot_act's first half); the actions go to the host, -1 for a slot not playing
//   observe   the host's rows (observation, reward, done, legal mask, to_play) -> host_observe_kernel: the rest of
//             record_move, fin, packing (pack_game, the step kernel's code), the stacked tail
//   restart   the next game's first rows of the slots observe packed -> host_start_kernel
// A finished game that does not fit into the staging area stays parked in its slot (fin > 0, action -1) and every
// observe pass tries again; the slot reports "finished" (its environment is reset, then restarted) once it is packed.
// mz_selfplay_begin_host_window: the caller keeps each game's observations.  rec_obs then holds a window of stack + 1
// rows per slot (observation p in row p % rows: all stack_fill reads) and the staged blocks carry none (O_staged = 0).
// Their test-mode games (mz_selfplay_begin_host_vs): after begin, observe and restart, the slots whose side to move is
// the opponent's play the opponent's move as a move of its own: opponent_turn (host_opponent_turn_kernel, the random
// default of opponent_move's draw) -> opponent_act (host_opponent_act_kernel: the host's or the default move, recorded
// with a NaN root and no visits) -> the host's step -> observe, which completes it as it completes MuZero's.
//
// User environments (MZ_ENV_USER, mz_selfplay_begin_user): the host-stepped loop's kernels with the host's step replaced
// by the wrapper kernels of a plug-in's CUDA source (user_env.cuh, compiled by user_env.cu), which write the rows the
// host would have uploaded.  A move is act -> mz_user_env_step -> observe -> mz_user_env_reset on the slots observe
// packed -> restart, all on the handle's stream (user_pass).
// Their test-mode games (mz_selfplay_begin_user_vs): a move is that pass for MuZero (host_act_kernel skips the slots whose
// side to move is the opponent's), then kUserOpponentPasses opponent passes: opponent_turn -> [mz_user_env_expert, the
// source's mz_env_expert, for MZ_OPPONENT_EXPERT] -> opponent_act -> the same step, observe, reset and restart; begin
// runs them too, so the opponent opens the games where it moves first.  The second pass plays the openings of the games
// the first pass's moves ended, so a game whose sides alternate is played in the moves the device environments' loop
// plays it in (that loop replies and opens in its step kernel), and finishes in the same call.  A slot whose opponent
// moves a third time in a row idles through the next search: every draw is keyed by game id and move, so its games
// do not change.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "handle.h"
#include "common.cuh"
#include "stack.cuh"
#include "user_env.cuh"

namespace mz {

constexpr int kMaxCells = 256;             // board cells per slot (Gomoku: up to 16 x 16)

struct SpDev {
    int env, B, A, O, H, W, K, max_moves, threshold, reward_scale;
    int O_in;                  // floats of a slot's search input: O, plus stack * (O + plane) stacked floats
    int stack;                 // config.stacked_observations
    int plane;                 // floats of one observation plane (the action plane of the stack has this size)
    int rows;                  // observations rec_obs keeps per slot: observation p of a game is row p % rows, with
                               // rows = max_moves + 1 (the whole game) or stack + 1 (a window: the caller keeps the game's)
    int O_staged;              // floats per observation in a staged block: O, or 0 for a window
    int opponent;              // MZ_OPPONENT_*
    int muzero_player;         // to_play of MuZero's side when opponent != MZ_OPPONENT_SELF
    uint64_t seed;
    int64_t id_stride;         // a slot's next game id = current + id_stride
    int td_steps;              // > 0: PER priorities are computed while packing (replay_buffer.py:33-51)
    double per_alpha;
    const double* discount_pow;   // [td_steps + 1] discount ** k as the caller's language evaluates it
    // environment state
    double* cart;              // [B][4]
    int* cart_steps;           // [B]
    int8_t* board;             // [B][kMaxCells], +1 / -1 / 0
    int8_t* player;            // [B] side to move, +1 / -1
    int32_t* ints;             // [B][4] Twenty-One: player's hand, dealer's hand, cards drawn; Simple Grid: row, column;
                               //        Gridworld: x, y, dir, step_count
    // search inputs / outputs (device)
    float* obs;                // [B][O_in]
    uint8_t* legal;            // [B][A]
    int32_t* to_play;          // [B]
    int64_t* game_id;          // [B]
    int32_t* move;             // [B] moves played in the current game
    int32_t* visits;           // [B][A]
    double* root_value;        // [B]
    // per-slot records of the game in flight
    double* rec_root;          // [B][T]
    int32_t* rec_visits;       // [B][T][A]
    int32_t* rec_action;       // [B][T]
    float* rec_reward;         // [B][T]
    int32_t* rec_to_play;      // [B][T]   (after the move)
    float* rec_obs;            // [B][rows][O]
    int32_t* first_to_play;    // [B]
    int32_t* fin;              // [B] 0 = playing, T > 0 = finished after T moves, waiting to be packed,
                               //     -1 = MZ_ENV_HOST: packed, waiting for the next game's first rows
    int32_t* last_action;      // [B]
    int32_t* host_action;      // [B] MZ_ENV_HOST / MZ_ENV_USER: the action of the move in flight, -1 for a slot not
                               //     playing it
    // counters: [0] env_steps, [1] games_finished, [2] staging cursor (may run past the capacity), [3] staged games,
    //           [4] park events of this call, [5] end of the valid staged bytes, [6] illegal opponent moves
    //           (MZ_ENV_HOST), [7] rows a user environment wrote that the loop could not play and illegal moves of its
    //           expert (MZ_ENV_USER)
    unsigned long long* counters;
    unsigned char* staging;    // mapped pinned host memory
    unsigned long long staging_cap;
    unsigned long long* index; // mapped pinned host memory: per staged game {byte offset, (slot << 32) | length}
    // per-move overrides (device copies) or nullptr
    const int32_t* forced_action;
    const double* uniform;
    double temperature;
};

// ------------------------------------------------------------------------------------------
// environments
// ------------------------------------------------------------------------------------------
constexpr double kGravity = 9.8, kMassCart = 1.0, kMassPole = 0.1, kHalfLen = 0.5, kForce = 10.0, kDt = 0.02;
constexpr double kXLimit = 2.4;
constexpr int kEpisodeCap = 500;

MZ_DEVINL void cartpole_reset(const SpDev& s, int g, int64_t gid) {
    double* st = s.cart + (size_t)g * 4;
    for (int k = 0; k < 4; ++k) {
        const double u = philox_uniform53(s.seed, gid, 0, (uint32_t)k, kTagReset);
        st[k] = -0.05 + 0.1 * u;                                   // uniform(-0.05, 0.05) like gym's reset
    }
    s.cart_steps[g] = 0;
}

MZ_DEVINL void cartpole_observe(const SpDev& s, int g, float* out) {
    const double* st = s.cart + (size_t)g * 4;
    for (int k = 0; k < 4; ++k) out[k] = (float)st[k];
}

// returns done; reward is always 1
MZ_DEVINL bool cartpole_step(const SpDev& s, int g, int action) {
    double* st = s.cart + (size_t)g * 4;
    const double x = st[0], xd = st[1], th = st[2], thd = st[3];
    const double force = action == 1 ? kForce : -kForce;
    const double c = cos(th), sn = sin(th);
    const double total = kMassCart + kMassPole, pml = kMassPole * kHalfLen;
    const double tmp = (force + pml * thd * thd * sn) / total;
    const double thacc = (kGravity * sn - c * tmp) / (kHalfLen * (4.0 / 3.0 - kMassPole * c * c / total));
    const double xacc = tmp - pml * thacc * c / total;
    st[0] = x + kDt * xd; st[1] = xd + kDt * xacc; st[2] = th + kDt * thd; st[3] = thd + kDt * thacc;
    const int steps = ++s.cart_steps[g];
    const double theta_limit = 12.0 * 2.0 * 3.141592653589793 / 360.0;
    return fabs(st[0]) > kXLimit || fabs(st[2]) > theta_limit || steps >= kEpisodeCap;
}

// Twenty-One: the slot's next card, 1 + floor(12 u) like randint(1, 13), face cards counting 10
MZ_DEVINL int twentyone_card(const SpDev& s, int g) {
    int32_t* st = s.ints + (size_t)g * 4;
    const double u = philox_uniform53(s.seed, s.game_id[g], st[2]++, 0u, kTagCard);
    const int card = 1 + (int)(12.0 * u);
    return card < 10 ? card : 10;
}

MZ_DEVINL void twentyone_reset(const SpDev& s, int g) {
    int32_t* st = s.ints + (size_t)g * 4;
    st[2] = 0;
    st[0] = twentyone_card(s, g);
    st[1] = twentyone_card(s, g);
}

// returns done; *reward = get_reward(done) * reward_scale
MZ_DEVINL bool twentyone_step(const SpDev& s, int g, int action, float* reward) {
    int32_t* st = s.ints + (size_t)g * 4;
    if (action == 0) st[0] += twentyone_card(s, g);
    const bool done = st[0] > 21 || action == 1 || st[0] == 21;
    int r = 0;
    if (done) {
        if (st[0] <= 21)
            while (st[1] <= 16) st[1] += twentyone_card(s, g);
        const int p = st[0], d = st[1];
        r = (p <= 21 && (d < p || d > 21)) ? 1 : (p > 21 ? -1 : (p == d ? 0 : -1));
    }
    *reward = (float)(r * s.reward_scale);
    return done;
}

// Simple Grid: returns done (the corner (2, 2) reached)
MZ_DEVINL bool grid_step(const SpDev& s, int g, int action) {
    int32_t* st = s.ints + (size_t)g * 4;
    if (action == 0 && st[0] < 2) ++st[0];
    if (action == 1 && st[1] < 2) ++st[1];
    return st[0] == 2 && st[1] == 2;
}

// Gridworld (games/gridworld.py): the agent on the floor(15 u0)-th free cell, x = 1 + i % 4, y = 1 + i / 4 (the goal
// would be i = 15; 15 u < 15 for every u < 1), facing floor(4 u1); u_k from draw k of the game's placement stream
MZ_DEVINL void gridworld_reset(const SpDev& s, int g, int64_t gid) {
    int32_t* st = s.ints + (size_t)g * 4;
    const int i = (int)(15.0 * philox_uniform53(s.seed, gid, 0, 0u, kTagPlace));
    st[0] = 1 + i % 4;
    st[1] = 1 + i / 4;
    st[2] = (int)(4.0 * philox_uniform53(s.seed, gid, 1, 0u, kTagPlace));
    st[3] = 0;
}

// the view [x'][y'][c]: view cell (x', y') lies 6 - y' cells ahead of the agent and x' - 3 cells to its right (the
// rules' window rotated dir + 1 times); cells outside the room read as walls, the agent's own cell (3, 6) as empty
MZ_DEVINL void gridworld_observe(const SpDev& s, int g, float* out) {
    const int32_t* st = s.ints + (size_t)g * 4;
    const int d = st[2];
    const int fx = d == 0 ? 1 : (d == 2 ? -1 : 0), fy = d == 1 ? 1 : (d == 3 ? -1 : 0);   // ahead; right = (-fy, fx)
#pragma unroll 1
    for (int xv = 0; xv < 7; ++xv)
#pragma unroll 1
        for (int yv = 0; yv < 7; ++yv) {
            const int ahead = 6 - yv, right = xv - 3;
            const int x = st[0] + ahead * fx - right * fy, y = st[1] + ahead * fy + right * fx;
            const bool own = xv == 3 && yv == 6;
            const bool wall = !own && (x <= 0 || x >= 5 || y <= 0 || y >= 5);
            const bool goal = !own && x == 4 && y == 4;
            float* c = out + (xv * 7 + yv) * 3;
            c[0] = wall ? 2.0f : (goal ? 8.0f : 1.0f);          // empty (1, 0, 0), wall (2, 5, 0), goal (8, 1, 0)
            c[1] = wall ? 5.0f : (goal ? 1.0f : 0.0f);
            c[2] = 0.0f;
        }
}

// returns done; *reward = 1 - 0.9 * (step_count / 144) in fp64 on entering the goal, rounded once to fp32
MZ_DEVINL bool gridworld_step(const SpDev& s, int g, int action, float* reward) {
    int32_t* st = s.ints + (size_t)g * 4;
    const int steps = ++st[3];
    const int d = st[2];
    bool goal = false;
    if (action == 0) {
        st[2] = (d + 3) & 3;
    } else if (action == 1) {
        st[2] = (d + 1) & 3;
    } else if (action == 2) {
        const int x = st[0] + (d == 0) - (d == 2), y = st[1] + (d == 1) - (d == 3);
        if (x >= 1 && x <= 4 && y >= 1 && y <= 4) { st[0] = x; st[1] = y; }
        goal = x == 4 && y == 4;
    }
    *reward = goal ? (float)(1.0 - 0.9 * ((double)steps / 144.0)) : 0.0f;
    return goal || steps >= 144;
}

MZ_DEVINL void board_reset(const SpDev& s, int g) {
    int8_t* b = s.board + (size_t)g * kMaxCells;
    for (int i = 0; i < kMaxCells; ++i) b[i] = 0;
    s.player[g] = 1;
}

MZ_DEVINL void board_observe(const SpDev& s, int g, float* out) {
    const int8_t* b = s.board + (size_t)g * kMaxCells;
    const int cells = s.H * s.W;
    const float side = (float)s.player[g];
    for (int i = 0; i < cells; ++i) {
        out[i] = b[i] == 1 ? 1.0f : 0.0f;
        out[cells + i] = b[i] == -1 ? 1.0f : 0.0f;
        out[2 * cells + i] = side;
    }
}

MZ_DEVINL void board_legal(const SpDev& s, int g, uint8_t* legal) {
    const int8_t* b = s.board + (size_t)g * kMaxCells;
    if (s.env == MZ_ENV_CONNECT4) {
        for (int x = 0; x < s.W; ++x) legal[x] = b[(s.H - 1) * s.W + x] == 0;
    } else {
        for (int i = 0; i < s.H * s.W; ++i) legal[i] = b[i] == 0;
    }
}

// places the mover's stone, returns (paid, done): paid = a line, or for Gomoku any end; the side to move flips
MZ_DEVINL void board_step(const SpDev& s, int g, int action, bool* paid, bool* done) {
    int8_t* b = s.board + (size_t)g * kMaxCells;
    const int me = s.player[g];
    int y = -1, x = -1;
    if (s.env == MZ_ENV_CONNECT4) {
        x = action;
        for (int r = 0; r < s.H; ++r) if (b[r * s.W + x] == 0) { y = r; break; }   // lowest empty row; a full column changes nothing
    } else {
        y = action / s.W; x = action % s.W;
    }
    bool w = false;
    if (y >= 0) {
        b[y * s.W + x] = (int8_t)me;
        // a new line must pass through the new stone
        const int dirs[4][2] = {{0, 1}, {1, 0}, {1, 1}, {-1, 1}};
        for (int d = 0; d < 4 && !w; ++d) {
            int run = 1;
            for (int sgn = -1; sgn <= 1; sgn += 2)
                for (int i = 1; i < s.K; ++i) {
                    const int yy = y + sgn * i * dirs[d][0], xx = x + sgn * i * dirs[d][1];
                    if (yy < 0 || yy >= s.H || xx < 0 || xx >= s.W || b[yy * s.W + xx] != me) break;
                    ++run;
                }
            w = run >= s.K;
        }
    }
    bool any = false;
    if (s.env == MZ_ENV_CONNECT4) { for (int c = 0; c < s.W; ++c) any |= b[(s.H - 1) * s.W + c] == 0; }
    else { for (int i = 0; i < s.H * s.W; ++i) any |= b[i] == 0; }
    s.player[g] = (int8_t)(-me);
    *paid = w || (s.env == MZ_ENV_GOMOKU && !any);
    *done = w || !any;
}

// writes the search inputs of slot g from its environment state (the current observation: the first O floats of the
// slot's input)
MZ_DEVINL void publish(const SpDev& s, int g) {
    float* o = s.obs + (size_t)g * s.O_in;
    uint8_t* lg = s.legal + (size_t)g * s.A;
    if (s.env == MZ_ENV_CARTPOLE || s.env == MZ_ENV_TWENTYONE || s.env == MZ_ENV_SIMPLE_GRID || s.env == MZ_ENV_GRIDWORLD) {
        const int32_t* st = s.ints + (size_t)g * 4;
        if (s.env == MZ_ENV_CARTPOLE) {
            cartpole_observe(s, g, o);
        } else if (s.env == MZ_ENV_GRIDWORLD) {
            gridworld_observe(s, g, o);
        } else if (s.env == MZ_ENV_TWENTYONE) {
            for (int i = 0; i < 9; ++i) { o[i] = (float)st[0]; o[9 + i] = (float)st[1]; o[18 + i] = 0.0f; }
        } else {
            for (int i = 0; i < 9; ++i) o[i] = i == st[0] * 3 + st[1] ? 1.0f : 0.0f;
        }
        for (int k = 0; k < s.A; ++k) lg[k] = 1;
        s.to_play[g] = 0;
    } else {
        board_observe(s, g, o);
        board_legal(s, g, lg);
        s.to_play[g] = s.player[g] == 1 ? 0 : 1;
    }
}

// numpy.random.choice(legal actions) for the uniform u: the legal action with index floor(u * n_legal), ascending
MZ_DEVINL int uniform_legal_pick(const uint8_t* lg, int A, double u) {
    int n_legal = 0, last = 0;
    for (int k = 0; k < A; ++k) if (lg[k]) { ++n_legal; last = k; }
    int idx = (int)(u * n_legal);
    if (idx >= n_legal) idx = n_legal - 1;
    for (int k = 0; k < A; ++k) if (lg[k] && idx-- == 0) return k;
    return last;
}

// ------------------------------------------------------------------------------------------
// the opponent of test-mode games (self_play.py:188-220)
// ------------------------------------------------------------------------------------------
// One window of the expert's scan (games/_boards.py::_threat_scan): `len` cells from (y0, x0) in steps (dy, dx).  A
// window whose stones sum to +-(len - 1) has one empty cell; its action becomes the candidate (a block, which a later
// window may overwrite) and returns true when the window is the mover's own (a win).  fixed >= 0: Connect4's vertical
// check, which names its column without looking at the gap.  Connect4 counts a gap only if it is the next free cell
// of its column (height = stones in the column, numpy.count_nonzero(board[:, x])).
MZ_DEVINL bool expert_window(const SpDev& s, const int8_t* b, int me, int y0, int x0, int dy, int dx, int len, int fixed,
                             int* action) {
    int sum = 0, gy = -1, gx = -1;
    for (int j = 0; j < len; ++j) {
        const int y = y0 + j * dy, x = x0 + j * dx;
        const int v = b[y * s.W + x];
        sum += v;
        if (v == 0 && gy < 0) { gy = y; gx = x; }
    }
    if (sum != len - 1 && sum != 1 - len) return false;
    if (fixed >= 0) {
        *action = fixed;
    } else if (s.env == MZ_ENV_CONNECT4) {
        int height = 0;
        for (int y = 0; y < s.H; ++y) height += b[y * s.W + gx] != 0;
        if (height != gy) return false;
        *action = gx;
    } else {
        *action = gy * s.W + gx;
    }
    return me * sum > 0;
}

// expert_action of games/tictactoe.py:308-349 and games/connect4.py:307-343 in their scan order; `dflt` is the random
// legal move the reference draws first
MZ_DEVINL int expert_action(const SpDev& s, int g, int dflt) {
    const int8_t* b = s.board + (size_t)g * kMaxCells;
    const int me = s.player[g];
    int a = dflt;
    if (s.env == MZ_ENV_TICTACTOE) {
        for (int i = 0; i < 3; ++i) {
            if (expert_window(s, b, me, i, 0, 0, 1, 3, -1, &a)) return a;       // row i
            if (expert_window(s, b, me, 0, i, 1, 0, 3, -1, &a)) return a;       // column i
        }
        if (expert_window(s, b, me, 0, 0, 1, 1, 3, -1, &a)) return a;           // diagonal
        if (expert_window(s, b, me, 0, 2, 1, -1, 3, -1, &a)) return a;          // numpy.fliplr(board).diagonal()
        return a;
    }
    for (int k = 0; k < 3; ++k)                                                  // 4x4 sub-board rows k.., columns l..
        for (int l = 0; l < 4; ++l) {
            for (int i = 0; i < 4; ++i) {
                if (expert_window(s, b, me, k + i, l, 0, 1, 4, -1, &a)) return a;
                if (expert_window(s, b, me, k, l + i, 1, 0, 4, l + i, &a)) return a;
            }
            if (expert_window(s, b, me, k, l, 1, 1, 4, -1, &a)) return a;
            if (expert_window(s, b, me, k, l + 3, 1, -1, 4, -1, &a)) return a;
        }
    return a;
}

// the opponent's move in slot g (legal mask published): the random legal default for the uniform u (or `dflt` when
// >= 0), improved by the expert's scan for MZ_OPPONENT_EXPERT
MZ_DEVINL int opponent_action(const SpDev& s, int g, double u, int dflt = -1) {
    const int d = dflt >= 0 ? dflt : uniform_legal_pick(s.legal + (size_t)g * s.A, s.A, u);
    return s.opponent == MZ_OPPONENT_EXPERT ? expert_action(s, g, d) : d;
}

// the search's part of the record of move t of slot g (store_search_statistics uses the pre-step root,
// self_play.py:169-175); root NaN and visits nullptr (all zero) mark a move no search chose
MZ_DEVINL void record_search(const SpDev& s, int g, int t, int action, double root, const int32_t* visits) {
    const size_t r = (size_t)g * s.max_moves + t;
    s.rec_root[r] = root;
    for (int k = 0; k < s.A; ++k) s.rec_visits[r * s.A + k] = visits ? visits[k] : 0;
    s.rec_action[r] = action;
}

// record of move t of slot g, then the slot's search inputs for the next move
MZ_DEVINL void record_move(const SpDev& s, int g, int t, int action, float reward, double root, const int32_t* visits) {
    const size_t r = (size_t)g * s.max_moves + t;
    record_search(s, g, t, action, root, visits);
    s.rec_reward[r] = reward;
    publish(s, g);
    s.rec_to_play[r] = s.to_play[g];
    const float* o = s.obs + (size_t)g * s.O_in;
    float* ro = s.rec_obs + ((size_t)g * s.rows + (t + 1) % s.rows) * s.O;
    for (int i = 0; i < s.O; ++i) ro[i] = o[i];
    s.move[g] = t + 1;
    s.last_action[g] = action;
}

// plays and records the opponent's move s.move[g] in slot g; returns done
MZ_DEVINL bool opponent_move(const SpDev& s, int g) {
    const int t = s.move[g];
    const double u = philox_uniform53(s.seed, s.game_id[g], t, 0u, kTagOpponent);
    const int action = opponent_action(s, g, u);
    bool paid, done;
    board_step(s, g, action, &paid, &done);
    record_move(s, g, t, action, paid ? (float)s.reward_scale : 0.0f, __longlong_as_double(0x7FF8000000000000ll), nullptr);
    return done;
}

// starts game gid in slot g; returns the moves played (1 when the opponent opens)
MZ_DEVINL int start_game(const SpDev& s, int g, int64_t gid) {
    s.game_id[g] = gid;
    s.move[g] = 0;
    s.fin[g] = 0;
    s.last_action[g] = -1;
    if (s.env == MZ_ENV_CARTPOLE) cartpole_reset(s, g, gid);
    else if (s.env == MZ_ENV_TWENTYONE) twentyone_reset(s, g);
    else if (s.env == MZ_ENV_SIMPLE_GRID) { s.ints[(size_t)g * 4] = 0; s.ints[(size_t)g * 4 + 1] = 0; }
    else if (s.env == MZ_ENV_GRIDWORLD) gridworld_reset(s, g, gid);
    else board_reset(s, g);
    publish(s, g);
    s.first_to_play[g] = s.to_play[g];
    const float* o = s.obs + (size_t)g * s.O_in;
    float* r0 = s.rec_obs + (size_t)g * s.rows * s.O;
    for (int i = 0; i < s.O; ++i) r0[i] = o[i];
    if (s.opponent == MZ_OPPONENT_SELF || s.to_play[g] == s.muzero_player) return 0;
    const bool done = opponent_move(s, g);
    if (done || s.move[g] >= s.max_moves) s.fin[g] = s.move[g];
    return 1;
}

// The stacked tail of slot g's search input, after its current observation (GameHistory.get_stacked_observations(-1),
// self_play.py:513-550), by stack_tail_element (stack.cuh) with t the moves played: observation p is rec_obs row
// p % rows and action_history[p + 1] is rec_action[p].
// Threads lane, lane + step, ... share the floats; the slot's records must be visible to all of them.
MZ_DEVINL void stack_fill(const SpDev& s, int g, int lane, int step) {
    const int t = s.move[g];
    float* tail = s.obs + (size_t)g * s.O_in + s.O;
    const float* rec = s.rec_obs + (size_t)g * s.rows * s.O;
    const int32_t* act = s.rec_action + (size_t)g * s.max_moves;
    const auto frame = [&](int p) { return rec + (size_t)(p % s.rows) * s.O; };
    const auto action = [&](int p) { return act[p]; };
    for (int i = lane; i < s.stack * (s.O + s.plane); i += step)
        tail[i] = stack_tail_element(i, t, s.O, s.plane, s.A, frame, action);
}

__global__ void selfplay_reset_kernel(const SpDev s, int64_t first_game_id) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= s.B) return;
    const int played = start_game(s, g, first_game_id + g);
    if (s.stack) stack_fill(s, g, 0, 1);
    if (played) atomicAdd(&s.counters[0], (unsigned long long)played);
}

// ------------------------------------------------------------------------------------------
// select_action (self_play.py:222-245) on the visit counts of the search that just finished, then Game.step
// ------------------------------------------------------------------------------------------
// kMaxA: the bound on |A| the cdf array is sized for
template <int kMaxA>
MZ_DEVINL int sample_action(const SpDev& s, int g, double temperature, double u) {
    const int32_t* v = s.visits + (size_t)g * s.A;
    const uint8_t* lg = s.legal + (size_t)g * s.A;
    const int A = s.A;
    if (temperature == 0.0) {                                  // numpy.argmax: the first maximum in action order
        int best = -1, arg = 0;
        for (int k = 0; k < A; ++k) if (lg[k] && v[k] > best) { best = v[k]; arg = k; }
        return arg;
    }
    if (isinf(temperature)) return uniform_legal_pick(lg, A, u);   // numpy.random.choice(actions)
    // numpy.random.choice(actions, p=p) with p = visit_counts ** (1 / T) / sum(...): cdf = p.cumsum(), cdf /= cdf[-1],
    // then the number of cdf entries <= u.  Illegal actions carry p = 0 and repeat the previous entry, so counting
    // over the whole action space lands on the same legal action; after the division the last entry is exactly 1 > u.
    // 1/T is 1, 2 or 4 for every reference schedule (games/*.py visit_softmax_temperature_fn): integer powers are exact
    const double inv = 1.0 / temperature;
    double total = 0.0;
    double p[kMaxA];
    for (int k = 0; k < A; ++k) {
        double x = lg[k] ? (double)v[k] : 0.0;
        if (inv == 2.0) x = x * x;
        else if (inv == 4.0) { x = x * x; x = x * x; }
        else if (inv != 1.0) x = pow(x, inv);
        p[k] = x;
        total += x;
    }
    double cdf = 0.0;
    for (int k = 0; k < A; ++k) {
        cdf = __dadd_rn(cdf, __ddiv_rn(p[k], total));
        p[k] = cdf;
    }
    int pick = 0;
    for (int k = 0; k < A; ++k) pick += __ddiv_rn(p[k], cdf) <= u;
    return pick;
}

// the action of move t in slot g: the injected one, else select_action's sample on the Philox uniform of (game, t)
// with the temperature threshold applied
template <int kMaxA>
MZ_DEVINL int choose_action(const SpDev& s, int g, int t) {
    int action = s.forced_action ? s.forced_action[g] : -1;
    if (action < 0) {
        const double T = (s.threshold == 0 || t + 1 < s.threshold) ? s.temperature : 0.0;
        const double u = s.uniform ? s.uniform[g] : philox_uniform53(s.seed, s.game_id[g], t, 0u, kTagAction);
        action = sample_action<kMaxA>(s, g, T, u);
    }
    return action;
}

// select_action + Game.step + record for slot g (one thread), then the opponent's reply in a test-mode game; returns
// the moves played
template <int kMaxA>
MZ_DEVINL int slot_act(const SpDev& s, int g) {
    const int t = s.move[g];
    const int action = choose_action<kMaxA>(s, g, t);
    float reward;
    bool done;
    if (s.env == MZ_ENV_CARTPOLE) {
        done = cartpole_step(s, g, action);
        reward = 1.0f;
    } else if (s.env == MZ_ENV_TWENTYONE) {
        done = twentyone_step(s, g, action, &reward);
    } else if (s.env == MZ_ENV_SIMPLE_GRID) {
        done = grid_step(s, g, action);
        reward = done ? (float)s.reward_scale : 0.0f;
    } else if (s.env == MZ_ENV_GRIDWORLD) {
        done = gridworld_step(s, g, action, &reward);
    } else {
        bool paid;
        board_step(s, g, action, &paid, &done);
        reward = paid ? (float)s.reward_scale : 0.0f;
    }
    record_move(s, g, t, action, reward, s.root_value[g], s.visits + (size_t)g * s.A);
    int played = 1;
    // len(action_history) <= max_moves (self_play.py:123) counts both sides' moves
    if (s.opponent != MZ_OPPONENT_SELF && !done && t + 1 < s.max_moves && s.to_play[g] != s.muzero_player) {
        done = opponent_move(s, g);
        ++played;
    }
    if (done || s.move[g] >= s.max_moves) s.fin[g] = s.move[g];
    return played;
}

__host__ __device__ inline unsigned long long staged_block_bytes(int T, int A, int O) {
    unsigned long long b = MZ_STAGED_HEADER_BYTES;
    b += (unsigned long long)T * 8;                 // root_value
    b += (unsigned long long)T * A * 4;             // visit counts
    b += (unsigned long long)T * 4 * 4;             // action, reward, to_play, priority
    b += (unsigned long long)(T + 1) * O * 4;       // observations
    return (b + 7) & ~7ull;
}

// ReplayBuffer.save_game's initial priority of position i of the finished game in slot g (replay_buffer.py:39-51 with
// compute_target_value, :230-262), in the reference's operation order on fp64:
//   value = (+/-)root_value[i + td] * discount**td           if i + td < T, else 0
//   value += (+/-)reward_history[i + 1 + k] * discount**k    for k = 0 .. td - 1 while i + 1 + k <= T
//   priority = |root_value[i] - value| ** alpha
// reward_history[j + 1] = the reward of move j; to_play_history[0] = first_to_play, [j + 1] = to_play after move j.
MZ_DEVINL float initial_priority(const SpDev& s, int g, int T, int i) {
    const size_t r = (size_t)g * s.max_moves;
    auto to_play_hist = [&](int j) { return j == 0 ? s.first_to_play[g] : s.rec_to_play[r + j - 1]; };
    const int td = s.td_steps;
    const int me = to_play_hist(i);
    double value = 0.0;
    if (i + td < T) {
        const double last = to_play_hist(i + td) == me ? s.rec_root[r + i + td] : -s.rec_root[r + i + td];
        value = __dmul_rn(last, s.discount_pow[td]);
    }
    for (int k = 0; k < td && i + k < T; ++k) {
        const double rew = (double)s.rec_reward[r + i + k];
        const double signed_rew = to_play_hist(i + k) == me ? rew : -rew;
        value = __dadd_rn(value, __dmul_rn(signed_rew, s.discount_pow[k]));
    }
    const double d = fabs(__dsub_rn(s.rec_root[r + i], value));
    return (float)(s.per_alpha == 1.0 ? d : __dsqrt_rn(d));
}

// Copies the finished game of slot g (T moves) into the staging area with the 32 lanes of one warp; returns false when
// it does not fit (the game stays parked in its slot, packed by a later pass after the host has drained).  Staging space
// is reserved with ONE atomicAdd per finished game (a compare-and-swap loop serialises hundreds of finishing warps per
// move): the cursor may run past the capacity, reservations that end beyond it are void, and since the cursor only
// grows the valid reservations are a contiguous prefix whose end is tracked in counters[5].
MZ_DEVINL bool pack_game(const SpDev& s, int g, int T, int lane) {
    const unsigned long long bytes = staged_block_bytes(T, s.A, s.O_staged);
    unsigned long long off = 0;
    int ok = 0;
    if (lane == 0) {
        off = atomicAdd(&s.counters[2], bytes);
        ok = off + bytes <= s.staging_cap;
        if (ok) {
            atomicMax(&s.counters[5], off + bytes);
            atomicAdd(&s.counters[1], 1ull);
            const unsigned long long i = atomicAdd(&s.counters[3], 1ull);
            s.index[2 * i] = off;
            s.index[2 * i + 1] = ((unsigned long long)(unsigned)g << 32) | (unsigned)T;
        } else {
            atomicAdd(&s.counters[4], 1ull);
        }
    }
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if (!ok) return false;
    off = ((unsigned long long)__shfl_sync(0xffffffffu, (unsigned)(off >> 32), 0) << 32) | __shfl_sync(0xffffffffu, (unsigned)off, 0);
    unsigned char* dst = s.staging + off;
    if (lane == 0) {
        *reinterpret_cast<int64_t*>(dst) = s.game_id[g];
        int32_t* hd = reinterpret_cast<int32_t*>(dst + 8);
        hd[0] = g; hd[1] = T; hd[2] = s.first_to_play[g]; hd[3] = s.O_staged; hd[4] = s.A; hd[5] = (int32_t)bytes;
    }
    unsigned char* p = dst + MZ_STAGED_HEADER_BYTES;
    const size_t r = (size_t)g * s.max_moves;
    {
        double* d = reinterpret_cast<double*>(p);
        for (int i = lane; i < T; i += 32) d[i] = s.rec_root[r + i];
        p += (size_t)T * 8;
    }
    {
        int32_t* d = reinterpret_cast<int32_t*>(p);
        for (int i = lane; i < T * s.A; i += 32) d[i] = s.rec_visits[r * s.A + i];
        p += (size_t)T * s.A * 4;
        d = reinterpret_cast<int32_t*>(p);
        for (int i = lane; i < T; i += 32) d[i] = s.rec_action[r + i];
        p += (size_t)T * 4;
        float* f = reinterpret_cast<float*>(p);
        for (int i = lane; i < T; i += 32) f[i] = s.rec_reward[r + i];
        p += (size_t)T * 4;
        d = reinterpret_cast<int32_t*>(p);
        for (int i = lane; i < T; i += 32) d[i] = s.rec_to_play[r + i];
        p += (size_t)T * 4;
        f = reinterpret_cast<float*>(p);
        for (int i = lane; i < T; i += 32) f[i] = s.td_steps > 0 ? initial_priority(s, g, T, i) : 0.0f;
        p += (size_t)T * 4;
        f = reinterpret_cast<float*>(p);
        const float* src = s.rec_obs + (size_t)g * s.rows * s.O;       // the whole game when O_staged > 0
        for (int i = lane; i < (T + 1) * s.O_staged; i += 32) f[i] = src[i];
    }
    __syncwarp();
    return true;
}

// One warp per slot, 32 slots per CTA.  act != 0: lane 0 plays the slot's move (sampling, environment step, record)
// unless the slot is parked; then, whatever `act`, a finished game is copied into the staging area by the whole warp and
// the slot starts its next game (act == 0 is the drain-only pass that re-packs games parked by an earlier call).  With
// stacked observations, a slot whose move was played or whose game restarted then rebuilds its stacked tail with the
// whole warp.
// kMaxA (128 or 256, the least that holds |A|) sizes the sampler's stack array, so the configurations of up to 128
// actions keep their stack frame.
constexpr int kStepThreads = 1024;

template <int kMaxA>
__global__ void __launch_bounds__(kStepThreads) selfplay_step_kernel(const SpDev s, int act) {
    __shared__ int s_active;
    if (threadIdx.x == 0) s_active = 0;
    __syncthreads();
    const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    int T = 0;
    int changed = 0;                                  // the slot's move count or records changed in this pass
    if (g < s.B) {
        if (lane == 0) {
            T = s.fin[g];
            if (act && T == 0) {
                atomicAdd(&s_active, slot_act<kMaxA>(s, g));
                T = s.fin[g];
                changed = 1;
            }
        }
        T = __shfl_sync(0xffffffffu, T, 0);
        __syncwarp();
    }
    if (T != 0 && pack_game(s, g, T, lane)) {
        if (lane == 0) {
            const int played = start_game(s, g, s.game_id[g] + s.id_stride);
            if (played) atomicAdd(&s_active, played);
        }
        changed = 1;
    }
    if (s.stack && g < s.B && __any_sync(0xffffffffu, changed)) {
        __syncwarp();                                 // lane 0's records and move count, visible to the warp
        stack_fill(s, g, lane, 32);
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_active) atomicAdd(&s.counters[0], (unsigned long long)s_active);
}

static void launch_selfplay_step(const SpDev& s, int act, cudaStream_t stream) {
    const int grid = (s.B * 32 + kStepThreads - 1) / kStepThreads;
    if (s.A <= 128) selfplay_step_kernel<128><<<grid, kStepThreads, 0, stream>>>(s, act);
    else selfplay_step_kernel<256><<<grid, kStepThreads, 0, stream>>>(s, act);
}

// ------------------------------------------------------------------------------------------
// MZ_ENV_HOST: the environment step is the host's
// ------------------------------------------------------------------------------------------
// device copies of what the host uploads for the whole batch
struct HostRows {
    float* obs;                // [B][O]
    float* reward;             // [B]
    uint8_t* done;             // [B]
    uint8_t* legal;            // [B][A]
    int32_t* to_play;          // [B]
};

// publish() of a host-stepped slot: its observation row becomes the current observation (the first O floats of the
// search input) and rec_obs row t % rows, its legal-mask row the slot's mask.  Threads tid, tid + nt, ... share the copies.
MZ_DEVINL void take_rows(const SpDev& s, const HostRows& h, int g, int t, int tid, int nt) {
    const float* src = h.obs + (size_t)g * s.O;
    float* o = s.obs + (size_t)g * s.O_in;
    float* ro = s.rec_obs + ((size_t)g * s.rows + t % s.rows) * s.O;
    for (int i = tid; i < s.O; i += nt) {
        const float v = src[i];
        o[i] = v;
        ro[i] = v;
    }
    for (int k = tid; k < s.A; k += nt) s.legal[(size_t)g * s.A + k] = h.legal[(size_t)g * s.A + k];
}

// threads per slot of the observe / restart kernels (one CTA per slot): a warp for small observations, more for image
// frames and deep stacks, whose copies would otherwise run on a few SMs
static int host_slot_threads(const SpDev& s) { return s.O_in + s.A > 4096 ? 256 : 32; }

// one thread per slot: the action of every playing slot (fin == 0) and its search records; -1 for the others
constexpr int kActThreads = 128;

template <int kMaxA>
__global__ void __launch_bounds__(kActThreads) host_act_kernel(const SpDev s) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    bool playing = false;
    if (g < s.B) {
        int action = -1;
        if (s.fin[g] == 0 && (s.opponent == MZ_OPPONENT_SELF || s.to_play[g] == s.muzero_player)) {
            const int t = s.move[g];
            action = choose_action<kMaxA>(s, g, t);
            record_search(s, g, t, action, s.root_value[g], s.visits + (size_t)g * s.A);
            playing = true;
        }
        s.host_action[g] = action;
    }
    const unsigned n = __popc(__ballot_sync(0xffffffffu, playing));
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&s.counters[0], (unsigned long long)n);
}

// One CTA per slot.  A slot that played finishes its move t with the host's rows (record_move's second half) and is
// finished when done or at max_moves; then every finished slot, parked ones included, is packed by warp 0.
// finished[g] = 1: the slot's game was packed in this pass and the slot waits for the next game's first rows (fin = -1).
__global__ void host_observe_kernel(const SpDev s, const HostRows h, uint8_t* finished) {
    __shared__ int s_T;
    const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int a = s.host_action[g];
    const int t = s.move[g];
    if (tid == 0) s_T = s.fin[g];
    __syncthreads();                                  // every thread has read the slot's state before it changes
    if (a >= 0) {
        take_rows(s, h, g, t + 1, tid, nt);
        if (tid == 0) {
            const size_t r = (size_t)g * s.max_moves + t;
            s.rec_reward[r] = h.reward[g];
            s.to_play[g] = h.to_play[g];
            s.rec_to_play[r] = h.to_play[g];
            s.move[g] = t + 1;
            s.last_action[g] = a;
            s_T = (h.done[g] || t + 1 >= s.max_moves) ? t + 1 : 0;
            s.fin[g] = s_T;
        }
    }
    __syncthreads();                                  // the records of move t, visible to the packing warp
    const int T = s_T;
    if (T > 0) {
        if (tid < 32) {
            const bool packed = pack_game(s, g, T, tid);
            if (tid == 0) {
                if (packed) s.fin[g] = -1;
                finished[g] = packed;
            }
        }
        return;
    }
    if (tid == 0) finished[g] = 0;
    if (a >= 0 && s.stack) stack_fill(s, g, tid, nt);
}

// One CTA per slot of `which` (all slots when nullptr, with the ids first_game_id + g): the slot starts a game from the
// host's first rows, as start_game does for the device environments.  A slot of `which` must be waiting (fin == -1).
__global__ void host_start_kernel(const SpDev s, const HostRows h, const uint8_t* which, int64_t first_game_id) {
    const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    if (which && !(which[g] && s.fin[g] == -1)) return;
    const int64_t gid = which ? s.game_id[g] + s.id_stride : first_game_id + g;
    __syncthreads();                                  // every thread has read the slot's state before it changes
    take_rows(s, h, g, 0, tid, nt);
    if (tid == 0) {
        s.game_id[g] = gid;
        s.move[g] = 0;
        s.fin[g] = 0;
        s.last_action[g] = -1;
        s.to_play[g] = h.to_play[g];
        s.first_to_play[g] = h.to_play[g];
    }
    __syncthreads();
    if (s.stack) stack_fill(s, g, tid, nt);
}

// Test-mode games of host-stepped environments (mz_selfplay_begin_host_vs): the opponent's move is a move of its own,
// stepped by the host between opponent_act and observe like MuZero's.  A slot's opponent move is due when its game is
// in play and the side to move is not MuZero's.
MZ_DEVINL bool opponent_due(const SpDev& s, int g) {
    return s.opponent != MZ_OPPONENT_SELF && s.fin[g] == 0 && s.to_play[g] != s.muzero_player;
}

// one thread per slot: the random default of every slot whose opponent move is due (opponent_move's draw on the
// published legal mask), -1 for the others
__global__ void __launch_bounds__(kActThreads) host_opponent_turn_kernel(const SpDev s, int32_t* defaults) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= s.B) return;
    int d = -1;
    if (opponent_due(s, g)) {
        const double u = philox_uniform53(s.seed, s.game_id[g], s.move[g], 0u, kTagOpponent);
        d = uniform_legal_pick(s.legal + (size_t)g * s.A, s.A, u);
    }
    defaults[g] = d;
}

// One thread per slot; `defaults` is the turn's (>= 0: the slot's opponent move is due), the move actions[g] or, when
// actions is nullptr, the default.  kCheck: count the due slots whose move is not legal in counters[6].  Otherwise, and
// only when that count is 0: record the move as opponent_move does (root NaN, no visit row), hand it to the host's step
// in host_action (-1 for the slots without one) and count it in env_steps.
template <bool kCheck>
__global__ void __launch_bounds__(kActThreads) host_opponent_act_kernel(const SpDev s, const int32_t* defaults,
                                                                        const int32_t* actions) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    bool moved = false;
    if (g < s.B) {
        const int d = defaults[g];
        const int a = d >= 0 && actions ? actions[g] : d;
        if (kCheck) {
            if (d >= 0 && (a < 0 || a >= s.A || !s.legal[(size_t)g * s.A + a])) atomicAdd(&s.counters[6], 1ull);
        } else if (s.counters[6] == 0) {
            if (d >= 0) record_search(s, g, s.move[g], a, __longlong_as_double(0x7FF8000000000000ll), nullptr);
            s.host_action[g] = a;
            moved = d >= 0;
        }
    }
    if (kCheck) return;
    const unsigned n = __popc(__ballot_sync(0xffffffffu, moved));
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&s.counters[0], (unsigned long long)n);
}

}  // namespace mz

using namespace mz;

// one thread per slot (the wrappers' __launch_bounds__); the expert wrapper takes the turn's defaults and writes actions
static cudaError_t launch_user_env(cudaKernel_t k, const MzUserEnvArgs& a, cudaStream_t stream,
                                   const int32_t* defaults = nullptr, int32_t* actions = nullptr) {
    void* args[] = {const_cast<MzUserEnvArgs*>(&a), &defaults, &actions};
    return cudaLaunchKernel(reinterpret_cast<const void*>(k), dim3((a.B + 127) / 128), dim3(128), args, 0, stream);
}

struct MzSelfPlay {
    MzSelfPlayDesc desc{};
    SpDev dev{};
    std::vector<void*> allocs;
    // two staging areas (pinned + mapped) used alternately: while the host reads the games of call i, call i+1 writes the
    // other one, so the copy on the host overlaps the next moves on the device
    unsigned char* staging[2] = {nullptr, nullptr};
    unsigned long long* index[2] = {nullptr, nullptr};
    unsigned char* d_staging[2] = {nullptr, nullptr};       // device views of the same memory
    unsigned long long* d_index[2] = {nullptr, nullptr};
    int cur = 0;                               // area the next mz_selfplay_moves / enqueue writes
    bool in_flight = false;                    // moves enqueued, not waited for yet
    unsigned long long* h_counters = nullptr;  // pinned copy of the counters
    int32_t* d_forced = nullptr;
    double* d_uniform = nullptr;
    double* d_noise = nullptr;
    int32_t* d_first = nullptr;
    uint64_t drained_bytes = 0;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    // MZ_ENV_HOST
    bool host = false;
    bool observe_due = false;                  // an act waits for its observe
    std::vector<int32_t> actions;              // the actions of the last act
    std::vector<uint8_t> awaiting;             // slots whose game was packed, waiting for mz_selfplay_host_restart
    int n_awaiting = 0;
    HostRows rows{};                           // device buffers of the host's uploads
    uint8_t* d_which = nullptr;
    uint8_t* d_finished = nullptr;
    float act_ms = 0.0f;
    // MZ_ENV_HOST test-mode games: 1 = begin, observe or restart ran and mz_selfplay_host_opponent_turn must look for
    // due opponent moves, 2 = it found some and they wait for mz_selfplay_host_opponent_act, 0 = MuZero moves next
    int opp_phase = 0;
    int32_t* d_defaults = nullptr;             // [B] the turn's random defaults, -1 for a slot without an opponent move
    int32_t* d_opp_actions = nullptr;          // [B] the host's opponent moves
    // MZ_ENV_USER: the rows and kernels of MZ_ENV_HOST, with the step and the reset on the device
    bool user = false;
    MzUserEnvKernels user_k{};
    MzUserEnvArgs user_args{};                 // the step's arguments; the reset's differ in `which`
};

void mz_selfplay_destroy(MzHandle* h) {
    if (!h || !h->sp) return;
    MzSelfPlay* sp = h->sp;
    for (void* p : sp->allocs) cudaFree(p);
    for (int i = 0; i < 2; ++i) {
        if (sp->staging[i]) cudaFreeHost(sp->staging[i]);
        if (sp->index[i]) cudaFreeHost(sp->index[i]);
    }
    if (sp->h_counters) cudaFreeHost(sp->h_counters);
    if (sp->e0) cudaEventDestroy(sp->e0);
    if (sp->e1) cudaEventDestroy(sp->e1);
    delete sp;
    h->sp = nullptr;
}

template <typename T>
static bool sp_alloc(MzSelfPlay* sp, T** p, size_t count) {
    void* q = nullptr;
    if (cudaMalloc(&q, count * sizeof(T) + 16) != cudaSuccess) return false;
    cudaMemset(q, 0, count * sizeof(T) + 16);
    sp->allocs.push_back(q);
    *p = reinterpret_cast<T*>(q);
    return true;
}

// The host's rows of a host-stepped batch: every row of `which` (all rows when nullptr) whose game goes on (`done` nullptr
// or 0) has a legal action, and every to_play names a player.  Returns MZ_OK or fails with the first bad row.
static int check_host_rows(MzHandle* h, const char* who, const uint8_t* which, const uint8_t* legal, const int32_t* to_play,
                           const uint8_t* done) {
    const int B = h->search.max_games, A = h->net.action_space, P = h->search.num_players;
    for (int g = 0; g < B; ++g) {
        if (which && !which[g]) continue;
        if (to_play[g] < 0 || to_play[g] >= P)
            return fail(h, MZ_EINVAL, std::string(who) + ": row " + std::to_string(g) + " has to_play " + std::to_string(to_play[g]) +
                                      ", outside the " + std::to_string(P) + " players");
        if (done && done[g]) continue;
        bool any = false;
        for (int k = 0; k < A && !any; ++k) any = legal[(size_t)g * A + k] != 0;
        if (!any) return fail(h, MZ_EINVAL, std::string(who) + ": row " + std::to_string(g) + " has no legal action");
    }
    return MZ_OK;
}

static int sp_begin(MzHandle* h, const MzSelfPlayDesc* d, int32_t opponent, int32_t muzero_player, const MzHostEnvDesc* e,
                    const float* obs, const uint8_t* legal, const int32_t* to_play, bool window,
                    const MzUserEnvDesc* u = nullptr, const MzUserEnvKernels* uk = nullptr);
enum { kUserPack = 0, kUserMuZero = 1, kUserOpponent = 2 };      // the passes of user_pass
constexpr int kUserOpponentPasses = 2;                            // opponent passes per move (and at begin)
static int user_pass(MzHandle* h, const SpDev& s, int pass);

extern "C" int mz_selfplay_begin(MzHandle* h, const MzSelfPlayDesc* d) {
    return mz_selfplay_begin_vs(h, d, MZ_OPPONENT_SELF, 0);
}

extern "C" int mz_selfplay_begin_vs(MzHandle* h, const MzSelfPlayDesc* d, int32_t opponent, int32_t muzero_player) {
    return sp_begin(h, d, opponent, muzero_player, nullptr, nullptr, nullptr, nullptr, false);
}

extern "C" int mz_selfplay_begin_host(MzHandle* h, const MzSelfPlayDesc* d, const MzHostEnvDesc* e, const float* obs,
                                      const uint8_t* legal, const int32_t* to_play) {
    if (!h || !d || !e || !obs || !legal || !to_play) return fail(h, MZ_EINVAL, "mz_selfplay_begin_host: null argument");
    if (d->env != MZ_ENV_HOST) return fail(h, MZ_EINVAL, "mz_selfplay_begin_host: desc->env must be MZ_ENV_HOST");
    return sp_begin(h, d, MZ_OPPONENT_SELF, 0, e, obs, legal, to_play, false);
}

extern "C" int mz_selfplay_begin_host_window(MzHandle* h, const MzSelfPlayDesc* d, const MzHostEnvDesc* e, const float* obs,
                                             const uint8_t* legal, const int32_t* to_play) {
    if (!h || !d || !e || !obs || !legal || !to_play) return fail(h, MZ_EINVAL, "mz_selfplay_begin_host_window: null argument");
    if (d->env != MZ_ENV_HOST) return fail(h, MZ_EINVAL, "mz_selfplay_begin_host_window: desc->env must be MZ_ENV_HOST");
    return sp_begin(h, d, MZ_OPPONENT_SELF, 0, e, obs, legal, to_play, true);
}

extern "C" int mz_selfplay_begin_host_vs(MzHandle* h, const MzSelfPlayDesc* d, const MzHostEnvDesc* e, int32_t opponent,
                                         int32_t muzero_player, int32_t window, const float* obs, const uint8_t* legal,
                                         const int32_t* to_play) {
    if (window != 0 && window != 1)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_host_vs: window must be 0 or 1, got " + std::to_string(window));
    if (opponent == MZ_OPPONENT_SELF && muzero_player == 0)
        return (window ? mz_selfplay_begin_host_window : mz_selfplay_begin_host)(h, d, e, obs, legal, to_play);
    if (!h || !d || !e || !obs || !legal || !to_play) return fail(h, MZ_EINVAL, "mz_selfplay_begin_host_vs: null argument");
    if (d->env != MZ_ENV_HOST) return fail(h, MZ_EINVAL, "mz_selfplay_begin_host_vs: desc->env must be MZ_ENV_HOST");
    return sp_begin(h, d, opponent, muzero_player, e, obs, legal, to_play, window == 1);
}

// window: rec_obs keeps the last stacked_observations + 1 observations of a slot's game and the staged blocks none
// (mz_selfplay_begin_host_window); otherwise the whole game's
// u, uk: the user environment of MZ_ENV_USER and its compiled kernels
static int sp_begin(MzHandle* h, const MzSelfPlayDesc* d, int32_t opponent, int32_t muzero_player, const MzHostEnvDesc* e,
                    const float* obs, const uint8_t* legal, const int32_t* to_play, bool window,
                    const MzUserEnvDesc* u, const MzUserEnvKernels* uk) {
    if (!h || !d) return fail(h, MZ_EINVAL, "mz_selfplay_begin: null argument");
    if (opponent != MZ_OPPONENT_SELF && opponent != MZ_OPPONENT_EXPERT && opponent != MZ_OPPONENT_RANDOM)
        return fail(h, MZ_EUNSUPPORTED, "mz_selfplay_begin_vs: unknown opponent " + std::to_string(opponent));
    if (opponent != MZ_OPPONENT_SELF && d->env == MZ_ENV_HOST && !e)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_vs: host-stepped games play against themselves only (test-mode games "
                                  "of host-stepped games begin with mz_selfplay_begin_host_vs)");
    if (opponent != MZ_OPPONENT_SELF && d->env == MZ_ENV_HOST && h->search.num_players < 2)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_host_vs: the handle's game has one player, its opponent is \"self\"");
    if (opponent != MZ_OPPONENT_SELF && d->env == MZ_ENV_USER && u && h->search.num_players < 2)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_user_vs: the handle's game has one player, its opponent is \"self\"");
    if (opponent == MZ_OPPONENT_EXPERT && d->env == MZ_ENV_USER && u && uk && !uk->expert)
        return fail(h, MZ_EUNSUPPORTED, "mz_selfplay_begin_user_vs: the source has no expert opponent: define MZ_ENV_EXPERT "
                                        "and __device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, "
                                        "const MzEnvRow& row, int default_action)");
    if (muzero_player != 0 && muzero_player != 1)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_vs: muzero_player must be 0 or 1, got " + std::to_string(muzero_player));
    if (opponent != MZ_OPPONENT_SELF && d->env == MZ_ENV_CARTPOLE)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_vs: CartPole has one player, its opponent is \"self\"");
    if (opponent != MZ_OPPONENT_SELF && (d->env == MZ_ENV_TWENTYONE || d->env == MZ_ENV_SIMPLE_GRID))
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_vs: Twenty-One and Simple Grid have one player, their opponent is \"self\"");
    if (opponent != MZ_OPPONENT_SELF && d->env == MZ_ENV_GRIDWORLD)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_vs: Gridworld has one player, its opponent is \"self\"");
    if (opponent == MZ_OPPONENT_EXPERT && d->env == MZ_ENV_GOMOKU)
        return fail(h, MZ_EUNSUPPORTED, "mz_selfplay_begin_vs: Gomoku has no expert opponent (the reference's Game has no expert_agent)");
    if (opponent != MZ_OPPONENT_SELF && d->td_steps > 0)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin_vs: test-mode games are not saved to a replay buffer, td_steps must be 0 "
                                  "(an opponent's move has no root value to bootstrap from)");
    if (d->stacked_observations < 0)
        return fail(h, MZ_EINVAL, "mz_selfplay_begin: stacked_observations must be >= 0, got " + std::to_string(d->stacked_observations));
    MZ_CUDA(h, cudaSetDevice(h->device));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    mz_selfplay_destroy(h);
    const int B = h->search.max_games, A = h->net.action_space;
    // board H x W and line length K; the observation's C planes of ph x pw; the action space
    int H = 1, W = 1, K = 0, C = 0, ph = 0, pw = 0, A_env = 0;
    const char* name = "";
    switch (d->env) {
        case MZ_ENV_CARTPOLE: name = "CartPole"; C = 1; ph = 1; pw = 4; A_env = 2; break;
        case MZ_ENV_TICTACTOE: name = "TicTacToe"; H = 3; W = 3; K = 3; C = 3; ph = 3; pw = 3; A_env = 9; break;
        case MZ_ENV_CONNECT4: name = "Connect4"; H = 6; W = 7; K = 4; C = 3; ph = 6; pw = 7; A_env = 7; break;
        case MZ_ENV_GOMOKU: {
            // the board's side is the reference's Gomoku.board_size; it travels in the handle's action space
            int side = 0;
            while ((side + 1) * (side + 1) <= A) ++side;
            if (side * side != A || side < 5 || side > 16)
                return fail(h, MZ_EINVAL, "mz_selfplay_begin: Gomoku plays on s x s boards with 5 <= s <= 16, so its action space is "
                                          "a square in [25, 256]; the handle has " + std::to_string(A) + " actions");
            name = "Gomoku"; H = side; W = side; K = 5; C = 3; ph = side; pw = side; A_env = A;
            break;
        }
        case MZ_ENV_TWENTYONE: name = "Twenty-One"; C = 3; ph = 3; pw = 3; A_env = 2; break;
        case MZ_ENV_SIMPLE_GRID: name = "Simple Grid"; C = 1; ph = 1; pw = 9; A_env = 2; break;
        // the reference's observation_shape (7, 7, 3): 7 planes of 7 x 3, the stack's planes too
        case MZ_ENV_GRIDWORLD: name = "Gridworld"; C = 7; ph = 7; pw = 3; A_env = 3; break;
        case MZ_ENV_HOST: {
            if (!e) return fail(h, MZ_EINVAL, "mz_selfplay_begin: host-stepped games (MZ_ENV_HOST) start with mz_selfplay_begin_host");
            if (e->obs_channels < 1 || e->obs_h < 1 || e->obs_w < 1)
                return fail(h, MZ_EINVAL, "mz_selfplay_begin_host: the observation's channels, height and width must be >= 1");
            int rc = check_host_rows(h, window ? "mz_selfplay_begin_host_window" : "mz_selfplay_begin_host", nullptr, legal,
                                     to_play, nullptr);
            if (rc) return rc;
            name = "the host-stepped environment"; C = e->obs_channels; ph = e->obs_h; pw = e->obs_w; A_env = A;
            break;
        }
        case MZ_ENV_USER: {
            if (!u || !uk) return fail(h, MZ_EINVAL, "mz_selfplay_begin: user environments (MZ_ENV_USER) start with mz_selfplay_begin_user");
            if (u->obs_channels < 1 || u->obs_h < 1 || u->obs_w < 1)
                return fail(h, MZ_EINVAL, "mz_selfplay_begin_user: the observation's channels, height and width must be >= 1");
            name = "the user environment"; C = u->obs_channels; ph = u->obs_h; pw = u->obs_w; A_env = A;
            break;
        }
        default: return fail(h, MZ_EUNSUPPORTED, "mz_selfplay_begin: unknown environment");
    }
    // the network input: the observation and, per stacked step, an earlier observation and its action plane
    const int64_t stack = d->stacked_observations, obs_c = (int64_t)C * (stack + 1) + stack;
    if (A != A_env || h->obs_elems != obs_c * ph * pw)
        return fail(h, MZ_EINVAL, std::string("mz_selfplay_begin: ") + name + " needs " + std::to_string(A_env) +
                                  " actions and, with stacked_observations = " + std::to_string(stack) + ", an input of obs_c = " +
                                  std::to_string(obs_c) + " planes of " + std::to_string(ph) + "x" + std::to_string(pw) +
                                  " (" + std::to_string(obs_c * ph * pw) + " values); the handle has " + std::to_string(A) +
                                  " actions and " + std::to_string(h->obs_elems) + " input values");
    const int O = C * ph * pw;
    if (d->max_moves < 1) return fail(h, MZ_EINVAL, "mz_selfplay_begin: max_moves < 1");
    // observations rec_obs keeps per slot, and the floats of each staged observation
    const int rows = window ? (int)stack + 1 : d->max_moves + 1, O_staged = window ? 0 : O;
    {
        // device memory per slot: the search input and outputs, the records of a maximum-length game (with `rows`
        // observations) and the host's upload rows
        const unsigned long long Tm = (unsigned long long)d->max_moves;
        const unsigned long long per_slot = (unsigned long long)h->obs_elems * 4 + (unsigned long long)rows * O * 4 +
                                            Tm * (8 + 4ull * A + 12) +
                                            (d->env == MZ_ENV_HOST || d->env == MZ_ENV_USER ? (unsigned long long)O * 4 + A + 16 : 0) +
                                            (d->env == MZ_ENV_USER ? (unsigned long long)u->state_bytes + 16 : 0) + 24ull * A + 64;
        size_t free_bytes = 0, total_bytes = 0;
        if (cudaMemGetInfo(&free_bytes, &total_bytes) == cudaSuccess && per_slot * B > free_bytes)
            return fail(h, MZ_ENOMEM, "mz_selfplay_begin: the records of " + std::to_string(B) + " slots do not fit on the device: " +
                                      std::to_string(per_slot) + " bytes per slot (" + (window ? "a window of " : "") +
                                      std::to_string(rows) + " observations of " + std::to_string(O) + " floats for max_moves = " +
                                      std::to_string(d->max_moves) + "), " + std::to_string(free_bytes) + " bytes free");
    }
    MzSelfPlay* sp = new (std::nothrow) MzSelfPlay();
    if (!sp) return fail(h, MZ_ENOMEM, "mz_selfplay_begin: out of host memory");
    h->sp = sp;
    sp->desc = *d;
    SpDev& s = sp->dev;
    s.env = d->env; s.B = B; s.A = A; s.O = O; s.H = H; s.W = W; s.K = K; s.max_moves = d->max_moves;
    s.O_in = (int)h->obs_elems; s.stack = (int)stack; s.plane = ph * pw; s.rows = rows; s.O_staged = O_staged;
    s.threshold = d->temperature_threshold; s.reward_scale = d->reward_scale; s.seed = h->search.seed;
    s.opponent = opponent; s.muzero_player = muzero_player;
    s.id_stride = d->game_id_stride > 0 ? d->game_id_stride : B;
    s.td_steps = 0; s.per_alpha = 1.0; s.discount_pow = nullptr;
    if (d->td_steps > 0) {
        if (!d->discount_pow || !(d->per_alpha == 0.5 || d->per_alpha == 1.0)) {
            mz_selfplay_destroy(h);
            return fail(h, MZ_EUNSUPPORTED, "mz_selfplay_begin: device priorities need discount_pow and per_alpha of 0.5 or 1");
        }
        double* dp = nullptr;
        if (!sp_alloc(sp, &dp, (size_t)d->td_steps + 1)) { mz_selfplay_destroy(h); return fail(h, MZ_ENOMEM, "mz_selfplay_begin: out of device memory"); }
        MZ_CUDA(h, cudaMemcpy(dp, d->discount_pow, ((size_t)d->td_steps + 1) * 8, cudaMemcpyHostToDevice));
        s.td_steps = d->td_steps; s.per_alpha = d->per_alpha; s.discount_pow = dp;
    }
    const size_t T = (size_t)d->max_moves;
    bool ok = sp_alloc(sp, &s.cart, (size_t)B * 4) && sp_alloc(sp, &s.cart_steps, B) && sp_alloc(sp, &s.board, (size_t)B * kMaxCells) &&
              sp_alloc(sp, &s.ints, (size_t)B * 4) &&
              sp_alloc(sp, &s.player, B) && sp_alloc(sp, &s.obs, (size_t)B * s.O_in) && sp_alloc(sp, &s.legal, (size_t)B * A) &&
              sp_alloc(sp, &s.to_play, B) && sp_alloc(sp, &s.game_id, B) && sp_alloc(sp, &s.move, B) &&
              sp_alloc(sp, &s.visits, (size_t)B * A) && sp_alloc(sp, &s.root_value, B) && sp_alloc(sp, &s.rec_root, B * T) &&
              sp_alloc(sp, &s.rec_visits, B * T * A) && sp_alloc(sp, &s.rec_action, B * T) && sp_alloc(sp, &s.rec_reward, B * T) &&
              sp_alloc(sp, &s.rec_to_play, B * T) && sp_alloc(sp, &s.rec_obs, B * (size_t)rows * O) && sp_alloc(sp, &s.first_to_play, B) &&
              sp_alloc(sp, &s.fin, B) && sp_alloc(sp, &s.last_action, B) && sp_alloc(sp, &s.counters, 8) &&
              sp_alloc(sp, &sp->d_forced, B) && sp_alloc(sp, &sp->d_uniform, B) && sp_alloc(sp, &sp->d_noise, (size_t)B * A) &&
              sp_alloc(sp, &sp->d_first, B) && sp_alloc(sp, &s.host_action, B);
    if (ok && (d->env == MZ_ENV_HOST || d->env == MZ_ENV_USER)) {
        float *r_obs = nullptr, *r_reward = nullptr;
        uint8_t *r_done = nullptr, *r_legal = nullptr;
        int32_t* r_to_play = nullptr;
        ok = sp_alloc(sp, &r_obs, (size_t)B * O) && sp_alloc(sp, &r_reward, B) && sp_alloc(sp, &r_done, B) &&
             sp_alloc(sp, &r_legal, (size_t)B * A) && sp_alloc(sp, &r_to_play, B) && sp_alloc(sp, &sp->d_which, B) &&
             sp_alloc(sp, &sp->d_finished, B) && sp_alloc(sp, &sp->d_defaults, B) && sp_alloc(sp, &sp->d_opp_actions, B);
        sp->rows = HostRows{r_obs, r_reward, r_done, r_legal, r_to_play};
        sp->host = d->env == MZ_ENV_HOST;
        sp->opp_phase = opponent != MZ_OPPONENT_SELF;
        sp->actions.assign(B, -1);
        sp->awaiting.assign(B, 0);
    }
    if (ok && d->env == MZ_ENV_USER) {
        MzUserEnvArgs& a = sp->user_args;
        a.state_stride = ((int64_t)u->state_bytes + 15) & ~(int64_t)15;
        ok = sp_alloc(sp, &a.state, (size_t)B * (a.state_stride > 0 ? a.state_stride : 1));
        a.B = B; a.O = O; a.A = A; a.P = h->search.num_players; a.seed = h->search.seed;
        a.game_id = s.game_id; a.move = s.move; a.action = s.host_action; a.which = sp->d_finished;
        a.first_game_id = d->first_game_id; a.id_stride = s.id_stride;
        a.obs = sp->rows.obs; a.reward = sp->rows.reward; a.done = sp->rows.done; a.legal = sp->rows.legal;
        a.to_play = sp->rows.to_play; a.bad = s.counters + 7;
        sp->user = true;
        sp->user_k = *uk;
    }
    if (!ok) { mz_selfplay_destroy(h); return fail(h, MZ_ENOMEM, "mz_selfplay_begin: out of device memory"); }
    // staging (two areas of this size): by default 4x the room for every slot finishing a maximum-length game at once,
    // within [16, 64] MiB;
    // whatever the size, games that do not fit wait in their slots (parked) - nothing is dropped
    unsigned long long cap = d->staging_bytes;
    const unsigned long long game_bytes = staged_block_bytes(d->max_moves, A, O_staged);
    if (cap == 0) {
        cap = 4 * game_bytes * (unsigned long long)B;
        if (cap < (16ull << 20)) cap = 16ull << 20;
        if (cap > (64ull << 20)) cap = 64ull << 20;
        if (cap < game_bytes) cap = game_bytes;
    }
    if (cap < game_bytes) { mz_selfplay_destroy(h); return fail(h, MZ_EINVAL, "mz_selfplay_begin: staging_bytes smaller than one game"); }
    const unsigned long long index_entries = cap / staged_block_bytes(1, A, O_staged) + 1;
    bool pinned = cudaHostAlloc(reinterpret_cast<void**>(&sp->h_counters), 64, cudaHostAllocDefault) == cudaSuccess;
    for (int i = 0; i < 2 && pinned; ++i)
        pinned = cudaHostAlloc(reinterpret_cast<void**>(&sp->staging[i]), cap, cudaHostAllocMapped) == cudaSuccess &&
                 cudaHostAlloc(reinterpret_cast<void**>(&sp->index[i]), index_entries * 16, cudaHostAllocMapped) == cudaSuccess;
    if (!pinned) {
        (void)cudaGetLastError();
        mz_selfplay_destroy(h);
        return fail(h, MZ_ENOMEM, "mz_selfplay_begin: pinned staging allocation failed");
    }
    memset(sp->h_counters, 0, 64);
    for (int i = 0; i < 2; ++i) {
        void* dptr = nullptr;
        if (cudaHostGetDevicePointer(&dptr, sp->staging[i], 0) != cudaSuccess) { mz_selfplay_destroy(h); return fail(h, MZ_ECUDA, "mz_selfplay_begin: staging is not device-mappable"); }
        sp->d_staging[i] = reinterpret_cast<unsigned char*>(dptr);
        if (cudaHostGetDevicePointer(&dptr, sp->index[i], 0) != cudaSuccess) { mz_selfplay_destroy(h); return fail(h, MZ_ECUDA, "mz_selfplay_begin: index is not device-mappable"); }
        sp->d_index[i] = reinterpret_cast<unsigned long long*>(dptr);
    }
    s.staging = sp->d_staging[0];
    s.index = sp->d_index[0];
    s.staging_cap = cap;
    cudaEventCreate(&sp->e0); cudaEventCreate(&sp->e1);
    if (sp->host || sp->user) {
        if (sp->host) {
            MZ_CUDA(h, cudaMemcpyAsync(sp->rows.obs, obs, (size_t)B * O * 4, cudaMemcpyHostToDevice, h->stream));
            MZ_CUDA(h, cudaMemcpyAsync(sp->rows.legal, legal, (size_t)B * A, cudaMemcpyHostToDevice, h->stream));
            MZ_CUDA(h, cudaMemcpyAsync(sp->rows.to_play, to_play, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
        } else {
            MzUserEnvArgs a = sp->user_args;
            a.which = nullptr;
            MZ_CUDA(h, launch_user_env(sp->user_k.reset, a, h->stream));
            h->launches += 1;
        }
        host_start_kernel<<<B, host_slot_threads(s), 0, h->stream>>>(s, sp->rows, nullptr, d->first_game_id);
        for (int p = 0; sp->user && opponent != MZ_OPPONENT_SELF && p < kUserOpponentPasses; ++p) {
            const int rc = user_pass(h, s, kUserOpponent);      // the opponent opens the games where it moves first
            if (rc) { mz_selfplay_destroy(h); return rc; }
        }
    } else {
        selfplay_reset_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(s, d->first_game_id);
    }
    h->launches += 1;
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    if (sp->user) {
        unsigned long long bad = 0;
        MZ_CUDA(h, cudaMemcpy(&bad, s.counters + 7, 8, cudaMemcpyDeviceToHost));
        if (bad) {
            mz_selfplay_destroy(h);
            if (opponent != MZ_OPPONENT_SELF)
                return fail(h, MZ_EINVAL, "mz_selfplay_begin_user_vs: the user environment's reset and the opponent's "
                                          "opening moves left " + std::to_string(bad) + " rows without a legal action or "
                                          "with a to_play outside the players, or expert moves that are not legal");
            return fail(h, MZ_EINVAL, "mz_selfplay_begin_user: mz_env_reset left " + std::to_string(bad) +
                                      " slots without a legal action or with a to_play outside the players");
        }
    }
    return MZ_OK;
}

static int sp_read_counters(MzHandle* h, MzSelfPlayStats* stats, float ms) {
    MzSelfPlay* sp = h->sp;
    MZ_CUDA(h, cudaMemcpyAsync(sp->h_counters, sp->dev.counters, 48, cudaMemcpyDeviceToHost, h->stream));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    if (stats) {
        stats->env_steps = (int64_t)sp->h_counters[0];
        stats->games_finished = (int64_t)sp->h_counters[1];
        stats->staged_bytes = (int64_t)sp->h_counters[5];
        stats->staged_games = (int32_t)sp->h_counters[3];
        stats->parked_slots = (int32_t)sp->h_counters[4];
        stats->device_ms = ms;
        stats->staging_capacity = (int64_t)sp->dev.staging_cap;
    }
    return MZ_OK;
}

// The kernel arguments of a move (the staging area in use, the temperature, the injected overrides copied to the
// device) and the search call on the slots' device-side inputs.
static int sp_move_setup(MzHandle* h, double temperature, const MzSelfPlayInject* inj, SpDev* out, SearchCall* call) {
    MzSelfPlay* sp = h->sp;
    SpDev& s = *out;
    s = sp->dev;
    s.staging = sp->d_staging[sp->cur];
    s.index = sp->d_index[sp->cur];
    const int B = s.B, A = s.A;
    s.temperature = temperature;
    s.forced_action = nullptr; s.uniform = nullptr;
    const double* noise = nullptr;
    const int32_t* first = nullptr;
    if (inj) {
        if (inj->forced_action) { MZ_CUDA(h, cudaMemcpyAsync(sp->d_forced, inj->forced_action, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream)); s.forced_action = sp->d_forced; }
        if (inj->uniform) { MZ_CUDA(h, cudaMemcpyAsync(sp->d_uniform, inj->uniform, (size_t)B * 8, cudaMemcpyHostToDevice, h->stream)); s.uniform = sp->d_uniform; }
        if (inj->noise) { MZ_CUDA(h, cudaMemcpyAsync(sp->d_noise, inj->noise, (size_t)B * A * 8, cudaMemcpyHostToDevice, h->stream)); noise = sp->d_noise; }
        if (inj->first_index) { MZ_CUDA(h, cudaMemcpyAsync(sp->d_first, inj->first_index, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream)); first = sp->d_first; }
    }
    *call = SearchCall{};
    call->n = B;
    call->obs = s.obs; call->legal_mask = s.legal; call->to_play = s.to_play;
    call->add_noise = 1; call->noise = noise; call->first_index = first;
    call->game_id = s.game_id; call->move_index = s.move;
    call->visit_counts = s.visits; call->root_value = s.root_value;
    return MZ_OK;
}

// One pass of a user environment's loop, then observe packs the finished games and their slots start the next game from
// the user reset's rows.  The pass's moves: kUserMuZero plays MuZero's (the act kernel on the search just run, then the
// user step on the slots that played), kUserOpponent the opponent's of the slots whose opponent move is due (its random
// default, improved by the source's expert for MZ_OPPONENT_EXPERT, recorded as host_opponent_act_kernel records, then the
// user step), kUserPack none: it only packs the games parked by an earlier call.
static int user_pass(MzHandle* h, const SpDev& s, int pass) {
    MzSelfPlay* sp = h->sp;
    const int B = s.B, grid = (B + kActThreads - 1) / kActThreads;
    if (pass == kUserMuZero) {
        if (s.A <= 128) host_act_kernel<128><<<grid, kActThreads, 0, h->stream>>>(s);
        else host_act_kernel<256><<<grid, kActThreads, 0, h->stream>>>(s);
        MZ_CUDA(h, launch_user_env(sp->user_k.step, sp->user_args, h->stream));
        h->launches += 2;
    } else if (pass == kUserOpponent) {
        const bool expert = s.opponent == MZ_OPPONENT_EXPERT;
        host_opponent_turn_kernel<<<grid, kActThreads, 0, h->stream>>>(s, sp->d_defaults);
        if (expert) MZ_CUDA(h, launch_user_env(sp->user_k.expert, sp->user_args, h->stream, sp->d_defaults, sp->d_opp_actions));
        host_opponent_act_kernel<false><<<grid, kActThreads, 0, h->stream>>>(s, sp->d_defaults, expert ? sp->d_opp_actions : nullptr);
        MZ_CUDA(h, launch_user_env(sp->user_k.step, sp->user_args, h->stream));
        h->launches += expert ? 4 : 3;
    } else {
        MZ_CUDA(h, cudaMemsetAsync(s.host_action, 0xFF, (size_t)B * 4, h->stream));     // -1: no slot plays
    }
    host_observe_kernel<<<B, host_slot_threads(s), 0, h->stream>>>(s, sp->rows, sp->d_finished);
    MZ_CUDA(h, launch_user_env(sp->user_k.reset, sp->user_args, h->stream));            // which = d_finished
    host_start_kernel<<<B, host_slot_threads(s), 0, h->stream>>>(s, sp->rows, sp->d_finished, 0);
    h->launches += 3;
    return MZ_OK;
}

static int sp_enqueue(MzHandle* h, int32_t n_moves, double temperature, const MzSelfPlayInject* inj, const char* who) {
    if (!h || !h->sp) return fail(h, MZ_ESTATE, std::string(who) + ": call mz_selfplay_begin first");
    if (!h->weights_loaded) return fail(h, MZ_ESTATE, std::string(who) + ": weights not loaded");
    if (n_moves < 0) return fail(h, MZ_EINVAL, std::string(who) + ": n_moves < 0");
    if (inj && n_moves > 1 && (inj->forced_action || inj->uniform || inj->noise || inj->first_index))
        return fail(h, MZ_EINVAL, std::string(who) + ": per-move overrides need n_moves == 1");
    if (!(temperature >= 0.0)) return fail(h, MZ_EINVAL, std::string(who) + ": temperature must be >= 0");
    MzSelfPlay* sp = h->sp;
    if (sp->host) return fail(h, MZ_ESTATE, std::string(who) + ": host-stepped games move with mz_selfplay_host_act / _observe / _restart");
    if (inj && inj->uniform)
        for (int g = 0; g < sp->dev.B; ++g)
            if (!(inj->uniform[g] >= 0.0 && inj->uniform[g] < 1.0))
                return fail(h, MZ_EINVAL, std::string(who) + ": injected uniforms must lie in [0, 1)");
    if (sp->in_flight) return fail(h, MZ_ESTATE, std::string(who) + ": moves already enqueued, call mz_selfplay_wait first");
    MZ_CUDA(h, cudaSetDevice(h->device));
    SpDev s;
    SearchCall call{};
    int rc = sp_move_setup(h, temperature, inj, &s, &call);
    if (rc) return rc;
    if (sp->drained_bytes) {
        // the host has taken the staged games (and the areas were swapped): rewind the cursor; parked games are packed
        // by the first pass below
        MZ_CUDA(h, cudaMemsetAsync(s.counters + 2, 0, 16, h->stream));
        MZ_CUDA(h, cudaMemsetAsync(s.counters + 5, 0, 8, h->stream));
        sp->drained_bytes = 0;
    }
    MZ_CUDA(h, cudaEventRecord(sp->e0, h->stream));
    if (sp->h_counters[4]) {                           // games parked by the previous call first, so their slots play again
        if (sp->user) {
            rc = user_pass(h, s, kUserPack);
            if (rc) return rc;
        } else {
            launch_selfplay_step(s, 0, h->stream);
            h->launches += 1;
        }
    }
    MZ_CUDA(h, cudaMemsetAsync(s.counters + 4, 0, 8, h->stream));      // [4] = park events of THIS call
    for (int m = 0; m < n_moves; ++m) {
        int rc = mz_dispatch_search(h, call, false, false, 0);
        if (rc) return rc;
        if (sp->user) {
            rc = user_pass(h, s, kUserMuZero);
            for (int p = 0; rc == MZ_OK && s.opponent != MZ_OPPONENT_SELF && p < kUserOpponentPasses; ++p)
                rc = user_pass(h, s, kUserOpponent);
            if (rc) return rc;
        } else {
            launch_selfplay_step(s, 1, h->stream);
            h->launches += 1;
        }
    }
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaEventRecord(sp->e1, h->stream));
    sp->in_flight = true;
    return MZ_OK;
}

static int sp_wait(MzHandle* h, MzSelfPlayStats* stats) {
    MzSelfPlay* sp = h->sp;
    int rc = sp_read_counters(h, stats, 0.0f);
    if (rc) return rc;
    sp->in_flight = false;
    if (h->res && resnet_take_saturations(h->res, h->stream) > 0) {
        // the moves above searched with towers outside their accuracy contract (activations beyond the fp16 range are
        // carried with a saturated high part, not dropped); later calls use the fp32 towers
        mz_switch_to_strict(h);
    }
    float ms = 0.0f;
    if (cudaEventElapsedTime(&ms, sp->e0, sp->e1) == cudaSuccess && stats) stats->device_ms = ms;
    if (sp->user) {
        MZ_CUDA(h, cudaMemcpy(sp->h_counters + 7, sp->dev.counters + 7, 8, cudaMemcpyDeviceToHost));
        if (sp->h_counters[7] && sp->dev.opponent == MZ_OPPONENT_EXPERT)
            return fail(h, MZ_EINVAL, "the user environment wrote " + std::to_string(sp->h_counters[7]) +
                                      " rows without a legal action or with a to_play outside the players (those games "
                                      "were ended there), or its mz_env_expert returned moves out of range or not legal "
                                      "(the random default was played instead); begin the loop again");
        if (sp->h_counters[7])
            return fail(h, MZ_EINVAL, "the user environment wrote " + std::to_string(sp->h_counters[7]) +
                                      " rows without a legal action or with a to_play outside the players (those games "
                                      "were ended there); begin the loop again");
    }
    return MZ_OK;
}

extern "C" int mz_selfplay_moves(MzHandle* h, int32_t n_moves, double temperature, const MzSelfPlayInject* inj, MzSelfPlayStats* stats) {
    if (h && h->sp && h->sp->user)
        return fail(h, MZ_ESTATE, "mz_selfplay_moves: a user environment's loop moves with mz_selfplay_user_moves");
    int rc = sp_enqueue(h, n_moves, temperature, inj, "mz_selfplay_moves");
    if (rc) return rc;
    return sp_wait(h, stats);
}

static int begin_user(MzHandle* h, const MzSelfPlayDesc* d, const MzUserEnvDesc* e, int32_t opponent, int32_t muzero_player,
                      const char* who) {
    if (!h || !d || !e || !e->source) return fail(h, MZ_EINVAL, std::string(who) + ": null argument");
    if (d->env != MZ_ENV_USER) return fail(h, MZ_EINVAL, std::string(who) + ": desc->env must be MZ_ENV_USER");
    if (e->state_bytes < 0 || e->state_bytes > MZ_USER_ENV_MAX_STATE_BYTES)
        return fail(h, MZ_EINVAL, std::string(who) + ": state_bytes must lie in [0, " +
                                  std::to_string(MZ_USER_ENV_MAX_STATE_BYTES) + "], got " + std::to_string(e->state_bytes));
    MZ_CUDA(h, cudaSetDevice(h->device));
    MzUserEnvKernels k;
    const int rc = mz_user_env_kernels(h, e->source, &k);
    if (rc) return rc;
    return sp_begin(h, d, opponent, muzero_player, nullptr, nullptr, nullptr, nullptr, false, e, &k);
}

extern "C" int mz_selfplay_begin_user(MzHandle* h, const MzSelfPlayDesc* d, const MzUserEnvDesc* e) {
    return begin_user(h, d, e, MZ_OPPONENT_SELF, 0, "mz_selfplay_begin_user");
}

extern "C" int mz_selfplay_begin_user_vs(MzHandle* h, const MzSelfPlayDesc* d, const MzUserEnvDesc* e, int32_t opponent,
                                         int32_t muzero_player) {
    if (opponent == MZ_OPPONENT_SELF && muzero_player == 0) return mz_selfplay_begin_user(h, d, e);
    return begin_user(h, d, e, opponent, muzero_player, "mz_selfplay_begin_user_vs");
}

extern "C" int mz_selfplay_user_moves(MzHandle* h, int32_t n_moves, double temperature, const MzSelfPlayInject* inj,
                                      MzSelfPlayStats* stats) {
    if (!h || !h->sp || !h->sp->user) return fail(h, MZ_ESTATE, "mz_selfplay_user_moves: call mz_selfplay_begin_user first");
    int rc = sp_enqueue(h, n_moves, temperature, inj, "mz_selfplay_user_moves");
    if (rc) return rc;
    return sp_wait(h, stats);
}

extern "C" int mz_selfplay_enqueue(MzHandle* h, int32_t n_moves, double temperature) {
    return sp_enqueue(h, n_moves, temperature, nullptr, "mz_selfplay_enqueue");
}

extern "C" int mz_selfplay_wait(MzHandle* h, MzSelfPlayStats* stats) {
    if (!h || !h->sp) return fail(h, MZ_ESTATE, "mz_selfplay_wait: call mz_selfplay_begin first");
    if (!h->sp->in_flight) return fail(h, MZ_ESTATE, "mz_selfplay_wait: nothing enqueued");
    MZ_CUDA(h, cudaSetDevice(h->device));
    return sp_wait(h, stats);
}

static int host_loop(MzHandle* h, const char* who) {
    if (!h || !h->sp || !h->sp->host) return fail(h, MZ_ESTATE, std::string(who) + ": call mz_selfplay_begin_host first");
    return MZ_OK;
}

extern "C" int mz_selfplay_host_act(MzHandle* h, double temperature, const MzSelfPlayInject* inj, int32_t* actions) {
    const char* who = "mz_selfplay_host_act";
    int rc = host_loop(h, who);
    if (rc) return rc;
    MzSelfPlay* sp = h->sp;
    if (!actions) return fail(h, MZ_EINVAL, std::string(who) + ": null actions");
    if (!h->weights_loaded) return fail(h, MZ_ESTATE, std::string(who) + ": weights not loaded");
    if (!(temperature >= 0.0)) return fail(h, MZ_EINVAL, std::string(who) + ": temperature must be >= 0");
    if (sp->observe_due) return fail(h, MZ_ESTATE, std::string(who) + ": the last act waits for mz_selfplay_host_observe");
    if (sp->n_awaiting)
        return fail(h, MZ_ESTATE, std::string(who) + ": " + std::to_string(sp->n_awaiting) +
                                  " finished slots wait for mz_selfplay_host_restart");
    if (sp->opp_phase == 1)
        return fail(h, MZ_ESTATE, std::string(who) + ": opponent moves may be due, call mz_selfplay_host_opponent_turn first");
    if (sp->opp_phase == 2)
        return fail(h, MZ_ESTATE, std::string(who) + ": opponent moves are due, call mz_selfplay_host_opponent_act first");
    const int B = sp->dev.B;
    if (inj && inj->uniform)
        for (int g = 0; g < B; ++g)
            if (!(inj->uniform[g] >= 0.0 && inj->uniform[g] < 1.0))
                return fail(h, MZ_EINVAL, std::string(who) + ": injected uniforms must lie in [0, 1)");
    MZ_CUDA(h, cudaSetDevice(h->device));
    SpDev s;
    SearchCall call{};
    rc = sp_move_setup(h, temperature, inj, &s, &call);
    if (rc) return rc;
    MZ_CUDA(h, cudaEventRecord(sp->e0, h->stream));
    rc = mz_dispatch_search(h, call, false, false, 0);
    if (rc) return rc;
    if (s.A <= 128) host_act_kernel<128><<<(B + kActThreads - 1) / kActThreads, kActThreads, 0, h->stream>>>(s);
    else host_act_kernel<256><<<(B + kActThreads - 1) / kActThreads, kActThreads, 0, h->stream>>>(s);
    h->launches += 1;
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaEventRecord(sp->e1, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(sp->actions.data(), s.host_action, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    if (h->res && resnet_take_saturations(h->res, h->stream) > 0) mz_switch_to_strict(h);    // as sp_wait
    sp->act_ms = 0.0f;
    cudaEventElapsedTime(&sp->act_ms, sp->e0, sp->e1);
    memcpy(actions, sp->actions.data(), (size_t)B * 4);
    sp->observe_due = true;
    return MZ_OK;
}

extern "C" int mz_selfplay_host_observe(MzHandle* h, const float* obs, const float* reward, const uint8_t* done,
                                        const uint8_t* legal, const int32_t* to_play, uint8_t* finished,
                                        MzSelfPlayStats* stats) {
    const char* who = "mz_selfplay_host_observe";
    int rc = host_loop(h, who);
    if (rc) return rc;
    MzSelfPlay* sp = h->sp;
    if (!obs || !reward || !done || !legal || !to_play || !finished) return fail(h, MZ_EINVAL, std::string(who) + ": null argument");
    if (!sp->observe_due) return fail(h, MZ_ESTATE, std::string(who) + ": no move in flight, call mz_selfplay_host_act first");
    const int B = sp->dev.B, A = sp->dev.A, O = sp->dev.O;
    std::vector<uint8_t> played(B);
    for (int g = 0; g < B; ++g) played[g] = sp->actions[g] >= 0;
    rc = check_host_rows(h, who, played.data(), legal, to_play, done);
    if (rc) return rc;
    MZ_CUDA(h, cudaSetDevice(h->device));
    const HostRows& r = sp->rows;
    MZ_CUDA(h, cudaMemcpyAsync(r.obs, obs, (size_t)B * O * 4, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(r.reward, reward, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(r.done, done, (size_t)B, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(r.legal, legal, (size_t)B * A, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(r.to_play, to_play, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
    SpDev s = sp->dev;
    s.staging = sp->d_staging[sp->cur];
    s.index = sp->d_index[sp->cur];
    if (sp->drained_bytes) {                       // as sp_enqueue: the host has taken the staged games
        MZ_CUDA(h, cudaMemsetAsync(s.counters + 2, 0, 16, h->stream));
        MZ_CUDA(h, cudaMemsetAsync(s.counters + 5, 0, 8, h->stream));
        sp->drained_bytes = 0;
    }
    MZ_CUDA(h, cudaMemsetAsync(s.counters + 4, 0, 8, h->stream));      // [4] = park events of THIS pass
    MZ_CUDA(h, cudaEventRecord(sp->e0, h->stream));
    host_observe_kernel<<<B, host_slot_threads(s), 0, h->stream>>>(s, r, sp->d_finished);
    h->launches += 1;
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaEventRecord(sp->e1, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(finished, sp->d_finished, (size_t)B, cudaMemcpyDeviceToHost, h->stream));
    rc = sp_read_counters(h, stats, 0.0f);         // synchronises
    if (rc) return rc;
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, sp->e0, sp->e1);
    if (stats) stats->device_ms = sp->act_ms + ms;
    for (int g = 0; g < B; ++g)
        if (finished[g]) { sp->awaiting[g] = 1; ++sp->n_awaiting; }
    sp->observe_due = false;
    sp->opp_phase = sp->dev.opponent != MZ_OPPONENT_SELF;
    return MZ_OK;
}

extern "C" int mz_selfplay_host_restart(MzHandle* h, const uint8_t* which, const float* obs, const uint8_t* legal,
                                        const int32_t* to_play) {
    const char* who = "mz_selfplay_host_restart";
    int rc = host_loop(h, who);
    if (rc) return rc;
    MzSelfPlay* sp = h->sp;
    if (!which || !obs || !legal || !to_play) return fail(h, MZ_EINVAL, std::string(who) + ": null argument");
    if (sp->observe_due) return fail(h, MZ_ESTATE, std::string(who) + ": the last act waits for mz_selfplay_host_observe");
    const int B = sp->dev.B, A = sp->dev.A, O = sp->dev.O;
    for (int g = 0; g < B; ++g)
        if (which[g] && !sp->awaiting[g])
            return fail(h, MZ_ESTATE, std::string(who) + ": slot " + std::to_string(g) +
                                      " has no packed game waiting for a restart (observe reports them as finished)");
    rc = check_host_rows(h, who, which, legal, to_play, nullptr);
    if (rc) return rc;
    MZ_CUDA(h, cudaSetDevice(h->device));
    const HostRows& r = sp->rows;
    MZ_CUDA(h, cudaMemcpyAsync(r.obs, obs, (size_t)B * O * 4, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(r.legal, legal, (size_t)B * A, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(r.to_play, to_play, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
    MZ_CUDA(h, cudaMemcpyAsync(sp->d_which, which, (size_t)B, cudaMemcpyHostToDevice, h->stream));
    host_start_kernel<<<B, host_slot_threads(sp->dev), 0, h->stream>>>(sp->dev, r, sp->d_which, 0);
    h->launches += 1;
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int g = 0; g < B; ++g)
        if (which[g]) { sp->awaiting[g] = 0; --sp->n_awaiting; }
    sp->opp_phase = sp->dev.opponent != MZ_OPPONENT_SELF;
    return MZ_OK;
}

// the opponent calls of a loop begun with mz_selfplay_begin_host_vs: MZ_ESTATE unless the loop has an opponent and is
// in the call's `phase` (opp_phase)
static int host_opponent_loop(MzHandle* h, const char* who, int phase) {
    int rc = host_loop(h, who);
    if (rc) return rc;
    MzSelfPlay* sp = h->sp;
    if (sp->dev.opponent == MZ_OPPONENT_SELF)
        return fail(h, MZ_ESTATE, std::string(who) + ": the loop plays against itself (begin it with mz_selfplay_begin_host_vs "
                                  "and an opponent)");
    if (sp->observe_due) return fail(h, MZ_ESTATE, std::string(who) + ": the last move waits for mz_selfplay_host_observe");
    if (sp->n_awaiting)
        return fail(h, MZ_ESTATE, std::string(who) + ": " + std::to_string(sp->n_awaiting) +
                                  " finished slots wait for mz_selfplay_host_restart");
    if (sp->opp_phase != phase)
        return fail(h, MZ_ESTATE, std::string(who) + (sp->opp_phase == 0 ? ": no opponent move is due, MuZero moves next (mz_selfplay_host_act)"
                                                      : sp->opp_phase == 1 ? ": call mz_selfplay_host_opponent_turn first"
                                                                           : ": opponent moves are due, call mz_selfplay_host_opponent_act"));
    MZ_CUDA(h, cudaSetDevice(h->device));
    return MZ_OK;
}

extern "C" int mz_selfplay_host_opponent_turn(MzHandle* h, int32_t* defaults) {
    const char* who = "mz_selfplay_host_opponent_turn";
    int rc = host_opponent_loop(h, who, 1);
    if (rc) return rc;
    if (!defaults) return fail(h, MZ_EINVAL, std::string(who) + ": null defaults");
    MzSelfPlay* sp = h->sp;
    const int B = sp->dev.B;
    host_opponent_turn_kernel<<<(B + kActThreads - 1) / kActThreads, kActThreads, 0, h->stream>>>(sp->dev, sp->d_defaults);
    h->launches += 1;
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaMemcpyAsync(defaults, sp->d_defaults, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    int due = 0;
    for (int g = 0; g < B; ++g) due += defaults[g] >= 0;
    sp->opp_phase = due ? 2 : 0;
    return due;
}

extern "C" int mz_selfplay_host_opponent_act(MzHandle* h, const int32_t* actions, int32_t* played) {
    const char* who = "mz_selfplay_host_opponent_act";
    int rc = host_opponent_loop(h, who, 2);
    if (rc) return rc;
    MzSelfPlay* sp = h->sp;
    if (!played) return fail(h, MZ_EINVAL, std::string(who) + ": null played");
    if (!actions && sp->dev.opponent == MZ_OPPONENT_EXPERT)
        return fail(h, MZ_EINVAL, std::string(who) + ": the EXPERT opponent's moves come from the host, actions is null");
    const int B = sp->dev.B;
    const SpDev& s = sp->dev;
    const int grid = (B + kActThreads - 1) / kActThreads;
    if (actions) MZ_CUDA(h, cudaMemcpyAsync(sp->d_opp_actions, actions, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
    const int32_t* d_actions = actions ? sp->d_opp_actions : nullptr;
    MZ_CUDA(h, cudaMemsetAsync(s.counters + 6, 0, 8, h->stream));
    host_opponent_act_kernel<true><<<grid, kActThreads, 0, h->stream>>>(s, sp->d_defaults, d_actions);
    host_opponent_act_kernel<false><<<grid, kActThreads, 0, h->stream>>>(s, sp->d_defaults, d_actions);
    h->launches += 2;
    MZ_CUDA(h, cudaGetLastError());
    MZ_CUDA(h, cudaMemcpyAsync(sp->h_counters + 6, s.counters + 6, 8, cudaMemcpyDeviceToHost, h->stream));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    if (sp->h_counters[6])                         // nothing was recorded: the opponent's moves can be given again
        return fail(h, MZ_EINVAL, std::string(who) + ": " + std::to_string(sp->h_counters[6]) +
                                  " opponent moves are not legal in their slot's published mask");
    MZ_CUDA(h, cudaMemcpy(sp->actions.data(), s.host_action, (size_t)B * 4, cudaMemcpyDeviceToHost));
    memcpy(played, sp->actions.data(), (size_t)B * 4);
    sp->act_ms = 0.0f;
    sp->opp_phase = 0;
    sp->observe_due = true;
    return MZ_OK;
}

extern "C" int mz_selfplay_drain(MzHandle* h, const void** data, uint64_t* bytes, int32_t* n_games, const uint64_t** index) {
    if (!h || !h->sp || !data || !bytes || !n_games) return fail(h, MZ_EINVAL, "mz_selfplay_drain: bad argument");
    MzSelfPlay* sp = h->sp;
    if (sp->in_flight) return fail(h, MZ_ESTATE, "mz_selfplay_drain: moves in flight, call mz_selfplay_wait first");
    MZ_CUDA(h, cudaSetDevice(h->device));
    if (sp->drained_bytes) {
        // drained already, and no move since has rewound the device's cursor: its counters still describe the games
        // returned then, from the other area
        *data = sp->staging[sp->cur];
        if (index) *index = reinterpret_cast<const uint64_t*>(sp->index[sp->cur]);
        *bytes = 0;
        *n_games = 0;
        return MZ_OK;
    }
    int rc = sp_read_counters(h, nullptr, 0.0f);
    if (rc) return rc;
    *data = sp->staging[sp->cur];
    if (index) *index = reinterpret_cast<const uint64_t*>(sp->index[sp->cur]);
    *bytes = sp->h_counters[5];
    *n_games = (int32_t)sp->h_counters[3];
    if (sp->h_counters[2]) {
        // the cursor moved (valid or void reservations): the next call rewinds it and writes the OTHER area, so what is
        // returned here stays intact while those moves run
        sp->drained_bytes = sp->h_counters[2];
        sp->cur ^= 1;
        sp->h_counters[2] = sp->h_counters[3] = sp->h_counters[5] = 0;     // a second drain before new moves returns nothing
    }
    return MZ_OK;
}

extern "C" int mz_selfplay_peek(MzHandle* h, const MzSelfPlayPeek* out) {
    if (!h || !h->sp || !out) return fail(h, MZ_EINVAL, "mz_selfplay_peek: bad argument");
    MZ_CUDA(h, cudaSetDevice(h->device));
    MZ_CUDA(h, cudaStreamSynchronize(h->stream));
    const SpDev& s = h->sp->dev;
    const size_t B = s.B;
    if (out->obs) MZ_CUDA(h, cudaMemcpy(out->obs, s.obs, B * s.O_in * 4, cudaMemcpyDeviceToHost));
    if (out->legal_mask) MZ_CUDA(h, cudaMemcpy(out->legal_mask, s.legal, B * s.A, cudaMemcpyDeviceToHost));
    if (out->to_play) MZ_CUDA(h, cudaMemcpy(out->to_play, s.to_play, B * 4, cudaMemcpyDeviceToHost));
    if (out->game_id) MZ_CUDA(h, cudaMemcpy(out->game_id, s.game_id, B * 8, cudaMemcpyDeviceToHost));
    if (out->move_index) MZ_CUDA(h, cudaMemcpy(out->move_index, s.move, B * 4, cudaMemcpyDeviceToHost));
    if (out->last_action) MZ_CUDA(h, cudaMemcpy(out->last_action, s.last_action, B * 4, cudaMemcpyDeviceToHost));
    return MZ_OK;
}

// debug: opponent_action over host positions, one thread per position
__global__ void opponent_debug_kernel(const SpDev s, const double* uniform, const int32_t* dflt, int32_t* out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= s.B) return;
    board_legal(s, g, s.legal + (size_t)g * s.A);
    out[g] = opponent_action(s, g, uniform ? uniform[g] : 0.0, dflt ? dflt[g] : -1);
}

extern "C" int mz_debug_opponent_action(int device, int32_t env, int32_t opponent, int32_t n, const int8_t* board,
                                        const int8_t* player, const double* uniform, const int32_t* default_action,
                                        int32_t* out) {
    SpDev s{};
    switch (env) {
        case MZ_ENV_TICTACTOE: s.H = 3; s.W = 3; s.K = 3; s.A = 9; break;
        case MZ_ENV_CONNECT4: s.H = 6; s.W = 7; s.K = 4; s.A = 7; break;
        case MZ_ENV_GOMOKU: s.H = 11; s.W = 11; s.K = 5; s.A = 121; break;
        default: return fail(nullptr, MZ_EUNSUPPORTED, "mz_debug_opponent_action: no opponent for this environment");
    }
    if (opponent != MZ_OPPONENT_EXPERT && opponent != MZ_OPPONENT_RANDOM)
        return fail(nullptr, MZ_EUNSUPPORTED, "mz_debug_opponent_action: opponent must be MZ_OPPONENT_EXPERT or MZ_OPPONENT_RANDOM");
    if (opponent == MZ_OPPONENT_EXPERT && env == MZ_ENV_GOMOKU)
        return fail(nullptr, MZ_EUNSUPPORTED, "mz_debug_opponent_action: Gomoku has no expert opponent");
    if (n < 1 || !board || !player || !out || (!uniform && !default_action))
        return fail(nullptr, MZ_EINVAL, "mz_debug_opponent_action: bad argument");
    const int cells = s.H * s.W;
    for (int i = 0; i < n; ++i) {
        if (player[i] != 1 && player[i] != -1) return fail(nullptr, MZ_EINVAL, "mz_debug_opponent_action: player must be +1 or -1");
        if (uniform && !(uniform[i] >= 0.0 && uniform[i] < 1.0)) return fail(nullptr, MZ_EINVAL, "mz_debug_opponent_action: uniforms must lie in [0, 1)");
        if (default_action && (default_action[i] < 0 || default_action[i] >= s.A))
            return fail(nullptr, MZ_EINVAL, "mz_debug_opponent_action: default action out of range");
        bool any = false;
        for (int c = 0; c < cells; ++c) {
            if (board[(size_t)i * cells + c] < -1 || board[(size_t)i * cells + c] > 1)
                return fail(nullptr, MZ_EINVAL, "mz_debug_opponent_action: board cells must be +1, -1 or 0");
            any |= board[(size_t)i * cells + c] == 0 && (env != MZ_ENV_CONNECT4 || c >= (s.H - 1) * s.W);
        }
        if (!any) return fail(nullptr, MZ_EINVAL, "mz_debug_opponent_action: a position without a legal action");
    }
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, MZ_ECUDA, "mz_debug_opponent_action: no such device");
    s.env = env; s.B = n; s.opponent = opponent;
    void* mem = nullptr;
    const size_t nb = (size_t)n * kMaxCells, np = (size_t)n, nl = (size_t)n * s.A, nu = (size_t)n * 8, nd = (size_t)n * 4, no = (size_t)n * 4;
    const size_t o_player = nb, o_legal = o_player + np, o_u = (o_legal + nl + 7) & ~(size_t)7, o_d = o_u + nu, o_out = o_d + nd;
    if (cudaMalloc(&mem, o_out + no) != cudaSuccess) { (void)cudaGetLastError(); return fail(nullptr, MZ_ENOMEM, "mz_debug_opponent_action: out of device memory"); }
    unsigned char* base = static_cast<unsigned char*>(mem);
    s.board = reinterpret_cast<int8_t*>(base);
    s.player = reinterpret_cast<int8_t*>(base + o_player);
    s.legal = base + o_legal;
    double* d_u = uniform ? reinterpret_cast<double*>(base + o_u) : nullptr;
    int32_t* d_d = default_action ? reinterpret_cast<int32_t*>(base + o_d) : nullptr;
    int32_t* d_out = reinterpret_cast<int32_t*>(base + o_out);
    cudaError_t e = cudaMemset(s.board, 0, nb);
    if (e == cudaSuccess) e = cudaMemcpy2D(s.board, kMaxCells, board, cells, cells, n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(s.player, player, np, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && d_u) e = cudaMemcpy(d_u, uniform, nu, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && d_d) e = cudaMemcpy(d_d, default_action, nd, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        opponent_debug_kernel<<<(n + 127) / 128, 128>>>(s, d_u, d_d, d_out);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, no, cudaMemcpyDeviceToHost);
    cudaFree(mem);
    if (e != cudaSuccess) return fail(nullptr, MZ_ECUDA, std::string("mz_debug_opponent_action: ") + cudaGetErrorString(e));
    return MZ_OK;
}
