"""Four built-in device environments of csrc/selfplay.cu restated as user environments (csrc/user_env.cuh): the sources a
plug-in would set as ``Game.DEVICE_SOURCE``.  Each must play the games of the built-in environment bit for bit
(tests/test_user_env_gpu.py); scripts/user_env_rate.py times two of them against it."""

# games/simple_grid.py: 3x3 grid from (0, 0), action 0 = row + 1, 1 = column + 1; 10 and done on reaching (2, 2)
SIMPLE_GRID = r"""
struct Grid { int row, col; };

__device__ void observe(const Grid* s, MzEnvRow& row) {
    for (int i = 0; i < 9; ++i) row.obs[i] = i == s->row * 3 + s->col ? 1.0f : 0.0f;
}

__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {
    Grid* s = static_cast<Grid*>(state);
    s->row = 0;
    s->col = 0;
    observe(s, row);
}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {
    Grid* s = static_cast<Grid*>(state);
    if (action == 0 && s->row < 2) ++s->row;
    if (action == 1 && s->col < 2) ++s->col;
    const bool done = s->row == 2 && s->col == 2;
    *row.reward = done ? 10.0f : 0.0f;
    *row.done = done;
    observe(s, row);
}
"""

# games/cartpole.py: Euler-integrated cart-pole, 20 ms step, +1 per step, done at |x| > 2.4, |theta| > 12 degrees or 500
# steps; the reset state from Philox draws (game id, 0, component, kTagReset) like the built-in environment's
CARTPOLE = r"""
struct Cart { double st[4]; int steps; };

__device__ void observe(const Cart* c, MzEnvRow& row) {
    for (int k = 0; k < 4; ++k) row.obs[k] = (float)c->st[k];
}

__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {
    Cart* c = static_cast<Cart*>(state);
    for (int k = 0; k < 4; ++k) c->st[k] = -0.05 + 0.1 * philox_uniform53(ctx.seed, ctx.game_id, 0, (uint32_t)k, kTagReset);
    c->steps = 0;
    observe(c, row);
}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {
    const double kGravity = 9.8, kMassCart = 1.0, kMassPole = 0.1, kHalfLen = 0.5, kForce = 10.0, kDt = 0.02;
    Cart* c = static_cast<Cart*>(state);
    double* st = c->st;
    const double x = st[0], xd = st[1], th = st[2], thd = st[3];
    const double force = action == 1 ? kForce : -kForce;
    const double cs = cos(th), sn = sin(th);
    const double total = kMassCart + kMassPole, pml = kMassPole * kHalfLen;
    const double tmp = (force + pml * thd * thd * sn) / total;
    const double thacc = (kGravity * sn - cs * tmp) / (kHalfLen * (4.0 / 3.0 - kMassPole * cs * cs / total));
    const double xacc = tmp - pml * thacc * cs / total;
    st[0] = x + kDt * xd; st[1] = xd + kDt * xacc; st[2] = th + kDt * thd; st[3] = thd + kDt * thacc;
    const int steps = ++c->steps;
    const double theta_limit = 12.0 * 2.0 * 3.141592653589793 / 360.0;
    *row.reward = 1.0f;
    *row.done = fabs(st[0]) > 2.4 || fabs(st[2]) > theta_limit || steps >= 500;
    observe(c, row);
}
"""

# games/gridworld.py: a 6x6 room, goal (4, 4), turn left / turn right / forward; the agent placed by Philox draws
# (game id, k, 0, kTagPlace); reward 1 - 0.9 * steps / 144 on reaching the goal, done there or at 144 steps; the 7x7x3
# egocentric view as 7 planes of 7 x 3
GRIDWORLD = r"""
struct Agent { int x, y, dir, steps; };

__device__ void observe(const Agent* a, MzEnvRow& row) {
    const int d = a->dir;
    const int fx = d == 0 ? 1 : (d == 2 ? -1 : 0), fy = d == 1 ? 1 : (d == 3 ? -1 : 0);
    for (int xv = 0; xv < 7; ++xv)
        for (int yv = 0; yv < 7; ++yv) {
            const int ahead = 6 - yv, right = xv - 3;
            const int x = a->x + ahead * fx - right * fy, y = a->y + ahead * fy + right * fx;
            const bool own = xv == 3 && yv == 6;
            const bool wall = !own && (x <= 0 || x >= 5 || y <= 0 || y >= 5);
            const bool goal = !own && x == 4 && y == 4;
            float* c = row.obs + (xv * 7 + yv) * 3;
            c[0] = wall ? 2.0f : (goal ? 8.0f : 1.0f);
            c[1] = wall ? 5.0f : (goal ? 1.0f : 0.0f);
            c[2] = 0.0f;
        }
}

__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {
    Agent* a = static_cast<Agent*>(state);
    const int i = (int)(15.0 * philox_uniform53(ctx.seed, ctx.game_id, 0, 0u, kTagPlace));
    a->x = 1 + i % 4;
    a->y = 1 + i / 4;
    a->dir = (int)(4.0 * philox_uniform53(ctx.seed, ctx.game_id, 1, 0u, kTagPlace));
    a->steps = 0;
    observe(a, row);
}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {
    Agent* a = static_cast<Agent*>(state);
    const int steps = ++a->steps;
    const int d = a->dir;
    bool goal = false;
    if (action == 0) {
        a->dir = (d + 3) & 3;
    } else if (action == 1) {
        a->dir = (d + 1) & 3;
    } else {
        const int x = a->x + (d == 0) - (d == 2), y = a->y + (d == 1) - (d == 3);
        if (x >= 1 && x <= 4 && y >= 1 && y <= 4) { a->x = x; a->y = y; }
        goal = x == 4 && y == 4;
    }
    *row.reward = goal ? (float)(1.0 - 0.9 * ((double)steps / 144.0)) : 0.0f;
    *row.done = goal || steps >= 144;
    observe(a, row);
}
"""

# games/tictactoe.py: two players, planes [stones of player +1, stones of player -1, side to move]; 20 to the mover on
# completing a line, done on a line or a full board; the legal mask is the empty cells
TICTACTOE = r"""
struct Board { int8_t cell[9]; int8_t player; };

__device__ void publish(const Board* b, MzEnvRow& row) {
    const float side = (float)b->player;
    for (int i = 0; i < 9; ++i) {
        row.obs[i] = b->cell[i] == 1 ? 1.0f : 0.0f;
        row.obs[9 + i] = b->cell[i] == -1 ? 1.0f : 0.0f;
        row.obs[18 + i] = side;
        row.legal[i] = b->cell[i] == 0;
    }
    *row.to_play = b->player == 1 ? 0 : 1;
}

__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {
    Board* b = static_cast<Board*>(state);
    for (int i = 0; i < 9; ++i) b->cell[i] = 0;
    b->player = 1;
    publish(b, row);
}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {
    Board* b = static_cast<Board*>(state);
    const int me = b->player, y = action / 3, x = action % 3;
    b->cell[action] = (int8_t)me;
    const int dirs[4][2] = {{0, 1}, {1, 0}, {1, 1}, {-1, 1}};
    bool line = false;
    for (int d = 0; d < 4 && !line; ++d) {
        int run = 1;
        for (int sgn = -1; sgn <= 1; sgn += 2)
            for (int i = 1; i < 3; ++i) {
                const int yy = y + sgn * i * dirs[d][0], xx = x + sgn * i * dirs[d][1];
                if (yy < 0 || yy >= 3 || xx < 0 || xx >= 3 || b->cell[yy * 3 + xx] != me) break;
                ++run;
            }
        line = run >= 3;
    }
    bool any = false;
    for (int i = 0; i < 9; ++i) any |= b->cell[i] == 0;
    b->player = (int8_t)(-me);
    *row.reward = line ? 20.0f : 0.0f;
    *row.done = line || !any;
    publish(b, row);
}
"""

# name -> (source, state bytes, the built-in environment's game module)
SOURCES = {
    "simple_grid": (SIMPLE_GRID, 8, "simple_grid"),
    "cartpole": (CARTPOLE, 40, "cartpole"),
    "gridworld": (GRIDWORLD, 16, "gridworld"),
    "tictactoe": (TICTACTOE, 10, "tictactoe"),
}
