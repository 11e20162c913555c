"""User environments with an expert opponent (csrc/user_env_expert.cuh): the sources test-mode games of the
"device-user-env" route play against.

* TICTACTOE and CONNECT4 restate the built-in device environments of csrc/selfplay.cu together with their expert
  (selfplay.cu's expert_action: games/tictactoe.py's and games/connect4.py's expert_agent in their scan order), so their
  test games must be the built-in environments' bit for bit.
* contract_expert_source / ExpertContractVector give the two-player cases of tests/user_env_contract_games.py one expert,
  written once in CUDA and once in Python, so their test games on the user route can be compared with the host-stepped
  route driven by the Python rules.
"""
import numpy

from user_env_contract_games import ContractVector, make_game
from user_env_sources import TICTACTOE as TICTACTOE_RULES

# A window of `len` cells from (y0, x0) in steps (dy, dx) whose stones sum to +-(len - 1) has one empty cell: its action
# becomes the candidate (a block, which a later window may overwrite) and the window ends the scan when it is the
# mover's own (a win).  Connect4 counts a gap only if it is the next free cell of its column, and its vertical windows
# name their column without looking at the gap.
TICTACTOE = TICTACTOE_RULES + r"""
#define MZ_ENV_EXPERT

__device__ bool expert_window(const Board* b, int y0, int x0, int dy, int dx, int* action) {
    int sum = 0, gy = -1, gx = -1;
    for (int j = 0; j < 3; ++j) {
        const int y = y0 + j * dy, x = x0 + j * dx, v = b->cell[y * 3 + x];
        sum += v;
        if (v == 0 && gy < 0) { gy = y; gx = x; }
    }
    if (sum != 2 && sum != -2) return false;
    *action = gy * 3 + gx;
    return b->player * sum > 0;
}

// rows and columns by index, then the diagonal and numpy.fliplr(board).diagonal()
__device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action) {
    const Board* b = static_cast<const Board*>(state);
    int a = default_action;
    for (int i = 0; i < 3; ++i) {
        if (expert_window(b, i, 0, 0, 1, &a)) return a;
        if (expert_window(b, 0, i, 1, 0, &a)) return a;
    }
    if (expert_window(b, 0, 0, 1, 1, &a)) return a;
    expert_window(b, 0, 2, 1, -1, &a);
    return a;
}
"""

# games/connect4.py: 6 rows x 7 columns, row 0 the bottom, actions are columns (a stone falls to the lowest empty row of
# its column); planes [stones of player +1, stones of player -1, side to move]; 10 to the mover on four in a row, done on
# a line or a full board; the legal mask is the columns whose top cell is empty
CONNECT4 = r"""
#define MZ_ENV_EXPERT

struct Board { int8_t cell[42]; int8_t player; };

__device__ void publish(const Board* b, MzEnvRow& row) {
    const float side = (float)b->player;
    for (int i = 0; i < 42; ++i) {
        row.obs[i] = b->cell[i] == 1 ? 1.0f : 0.0f;
        row.obs[42 + i] = b->cell[i] == -1 ? 1.0f : 0.0f;
        row.obs[84 + i] = side;
    }
    for (int x = 0; x < 7; ++x) row.legal[x] = b->cell[35 + x] == 0;
    *row.to_play = b->player == 1 ? 0 : 1;
}

__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {
    Board* b = static_cast<Board*>(state);
    for (int i = 0; i < 42; ++i) b->cell[i] = 0;
    b->player = 1;
    publish(b, row);
}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {
    Board* b = static_cast<Board*>(state);
    const int me = b->player, x = action;
    int y = -1;
    for (int r = 0; r < 6; ++r) if (b->cell[r * 7 + x] == 0) { y = r; break; }
    bool line = false;
    if (y >= 0) {
        b->cell[y * 7 + x] = (int8_t)me;
        const int dirs[4][2] = {{0, 1}, {1, 0}, {1, 1}, {-1, 1}};
        for (int d = 0; d < 4 && !line; ++d) {
            int run = 1;
            for (int sgn = -1; sgn <= 1; sgn += 2)
                for (int i = 1; i < 4; ++i) {
                    const int yy = y + sgn * i * dirs[d][0], xx = x + sgn * i * dirs[d][1];
                    if (yy < 0 || yy >= 6 || xx < 0 || xx >= 7 || b->cell[yy * 7 + xx] != me) break;
                    ++run;
                }
            line = run >= 4;
        }
    }
    bool any = false;
    for (int c = 0; c < 7; ++c) any |= b->cell[35 + c] == 0;
    b->player = (int8_t)(-me);
    *row.reward = line ? 10.0f : 0.0f;
    *row.done = line || !any;
    publish(b, row);
}

// -1: no candidate; else the window's action a as 2 * a + 1 for the mover's own line (a win), 2 * a for a block
__device__ int expert_window(const Board* b, int y0, int x0, int dy, int dx, int fixed) {
    int sum = 0, gy = -1, gx = -1;
    for (int j = 0; j < 4; ++j) {
        const int y = y0 + j * dy, x = x0 + j * dx, v = b->cell[y * 7 + x];
        sum += v;
        if (v == 0 && gy < 0) { gy = y; gx = x; }
    }
    if (sum != 3 && sum != -3) return -1;
    if (fixed < 0) {
        int height = 0;
        for (int y = 0; y < 6; ++y) height += b->cell[y * 7 + gx] != 0;
        if (height != gy) return -1;
    }
    return 2 * (fixed >= 0 ? fixed : gx) + (b->player * sum > 0);
}

// the 4x4 sub-boards at rows k.., columns l..: their rows and columns by index, then the diagonal and the anti-diagonal
__device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action) {
    const Board* b = static_cast<const Board*>(state);
    int a = default_action;
    for (int k = 0; k < 3; ++k)
        for (int l = 0; l < 4; ++l)
            for (int w = 0; w < 10; ++w) {
                const int i = w >> 1;
                const int c = w < 8 ? ((w & 1) ? expert_window(b, k, l + i, 1, 0, l + i) : expert_window(b, k + i, l, 0, 1, -1))
                                    : (w == 8 ? expert_window(b, k, l, 1, 1, -1) : expert_window(b, k, l + 3, 1, -1, -1));
                if (c < 0) continue;
                a = c >> 1;
                if (c & 1) return a;
            }
    return a;
}
"""

# name -> (source, state bytes, the built-in environment's game module)
SOURCES = {
    "tictactoe": (TICTACTOE, 10, "tictactoe"),
    "connect4": (CONNECT4, 43, "connect4"),
}

# An expert of no game, for the contract cases: it reads the state, the context and the published row (mask, to_play)
# and falls back to the library's default on some moves.  r = (resets of the slot + move + game id % 7 + to_play) % 3:
# 0 the default, 1 the highest legal action, 2 legal action move % (legal actions) in ascending order.
CONTRACT_EXPERT = r"""
#define MZ_ENV_EXPERT

__device__ int mz_env_expert(const void* state, const MzEnvCtx& ctx, const MzEnvRow& row, int default_action) {
    int count = 0;
#if MZ_SB > 0
    count = static_cast<const unsigned char*>(state)[0];
#endif
    const int r = (count + ctx.move + (int)(ctx.game_id % 7) + *row.to_play) % 3;
    if (r == 0) return default_action;
    int n = 0, last = -1;
    for (int a = 0; a < MZ_A; ++a) if (row.legal[a]) { ++n; last = a; }
    if (r == 1) return last;
    int i = ctx.move % n;
    for (int a = 0; a < MZ_A; ++a) if (row.legal[a] && i-- == 0) return a;
    return last;
}
"""


def contract_expert_source(case):
    return case.source + CONTRACT_EXPERT


class ExpertContractVector(ContractVector):
    """ContractVector with CONTRACT_EXPERT in Python (the host-stepped route's ``expert_actions``)."""

    def expert_actions(self, defaults, which):
        out = numpy.full(self.num_games, -1, numpy.int32)
        for g in numpy.nonzero(which)[0]:
            row = self.rows[g]
            count = int(self.state[g][0]) if self.case.state_bytes else 0
            r = (count + self.move[g] + self.gid[g] % 7 + int(row.to_play)) % 3
            legal = numpy.nonzero(row.legal)[0]
            out[g] = int(defaults[g]) if r == 0 else (int(legal[-1]) if r == 1 else int(legal[self.move[g] % len(legal)]))
        return out


def make_expert_game(case, first_game_id, stride, user=True):
    """make_game's plug-in with the contract expert: the CUDA one in ``DEVICE_SOURCE``, the Python one in ``vector``."""
    base = make_game(case, first_game_id, stride, user)

    class ExpertContractGame(base):
        DEVICE_SOURCE = contract_expert_source(case) if user else None

        @classmethod
        def vector(cls, num_games, seed=None):
            return ExpertContractVector(case, num_games, seed, first_game_id, stride)

    return ExpertContractGame
