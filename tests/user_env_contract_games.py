"""Test-only plug-in games that reach every edge of the user-environment contract (csrc/user_env.cuh), each with a
plain Python restatement of its rules.

Every case is one CUDA source for ``Game.DEVICE_SOURCE``, generated from one template by the case's sizes, and the same
rules on numpy: float32 arithmetic for the source's fp32, Python floats for its fp64, and ``oracle.philox.uniform53``
with the family's own tag for every random draw.  The rules:

* reset: byte 0 of the slot's state counts the slot's resets (the state persists across games); the observation is
  written; on three games in four the legal mask and to_play are written too (else the contract's defaults stay: every
  action legal, player 0).  A two-player game opens with player 1 about half the time.
* step (move m, draws at k = m + 1): every byte of the state is read (as 16-byte vectors, then a scalar tail) and bytes
  1.. are rewritten; reward ``-2 + 4u`` (both signs, not integers) and done are written; on one move in five nothing
  else (the previous move's observation, mask and to_play stay); else the observation, a new mask (one legal action on
  a quarter of the moves; on half of the terminal rows no legal action at all) and, for two players, the next player -
  the same player again on 30 % of the moves.
* a game's planned length L = 1 + floor(u * (max_moves + 2)) is drawn from its id: L = 1 ends on the first move,
  L = max_moves ends at exactly max_moves, L > max_moves is cut by max_moves while the environment goes on.
* the observation holds ctx.slot, ctx.move, ctx.game_id, the reset count, a checksum of every state byte, an fp32
  ``a * b + c`` and the bit pattern of an fp64 ``x * y + z`` (operands in [1, 2), where the fused and unfused results
  differ on some draws), the action, and a pattern of (k, game id) in the remaining floats.

A finished game is replayed from its record alone: slot and the slot's game count follow from ``first_game_id`` and
``game_id_stride`` (>= B), and a slot's games are replayed in order, so its state is rebuilt without knowing how the
device scheduled the slots.
"""
import math
import struct
from dataclasses import dataclass
from fractions import Fraction

import numpy

from muzero_general_b200.games._config import BaseMuZeroConfig
from muzero_general_b200.games.abstract_game import AbstractGame, VectorGame
from oracle.philox import uniform53

TAG = 0x7169E0C1          # the family's own Philox stream tag

SOURCE_TEMPLATE = r"""
#define MZ_A {A}
#define MZ_O {O}
#define MZ_P {P}
#define MZ_SB {SB}
#define MZ_LMAX {LMAX}
#define MZ_TAG {TAG}u

__device__ double draw(const MzEnvCtx& ctx, int k, unsigned c2) {{
    return philox_uniform53(ctx.seed, ctx.game_id, k, c2, MZ_TAG);
}}

// reads every state byte (16-byte vectors, then the tail) and returns sum (i + 1) * byte[i]; add >= 0 also rewrites
// bytes i >= 1 as byte + add + i
__device__ unsigned state_pass(unsigned char* s, int add) {{
    unsigned sum = 0;
    int i = 0;
#if MZ_SB >= 16
    for (; i + 16 <= MZ_SB; i += 16) {{
        const uint4 v = *reinterpret_cast<const uint4*>(s + i);
        unsigned w[4] = {{v.x, v.y, v.z, v.w}};
#pragma unroll
        for (int j = 0; j < 16; ++j) {{
            const int sh = 8 * (j & 3);
            unsigned b = (w[j >> 2] >> sh) & 255u;
            sum += b * (unsigned)(i + j + 1);
            if (add >= 0 && i + j >= 1) b = (b + (unsigned)(add + i + j)) & 255u;
            w[j >> 2] = (w[j >> 2] & ~(255u << sh)) | (b << sh);
        }}
        if (add >= 0) *reinterpret_cast<uint4*>(s + i) = make_uint4(w[0], w[1], w[2], w[3]);
    }}
#endif
    for (; i < MZ_SB; ++i) {{
        const unsigned b = s[i];
        sum += b * (unsigned)(i + 1);
        if (add >= 0 && i >= 1) s[i] = (unsigned char)(b + (unsigned)(add + i));
    }}
    return sum;
}}

__device__ void observe(const MzEnvCtx& ctx, MzEnvRow& row, int k, int action, int count, unsigned sum) {{
    float* o = row.obs;
    o[0] = (float)ctx.slot;
    o[1] = (float)ctx.move;
    o[2] = (float)(ctx.game_id & 0xFFFFF);
    o[3] = (float)(ctx.game_id >> 20);
    o[4] = (float)count;
    o[5] = (float)(sum & 0xFFFFu);
    o[6] = (float)(sum >> 16);
    const float a = (float)(1.0 + draw(ctx, k, 8)), b = (float)(1.0 + draw(ctx, k, 9)), c = (float)(1.0 + draw(ctx, k, 10));
    o[7] = a * b + c;
    const double x = 1.0 + draw(ctx, k, 11), y = 1.0 + draw(ctx, k, 12), z = 1.0 + draw(ctx, k, 13);
    const double d = x * y + z;
    const unsigned long long bits = (unsigned long long)__double_as_longlong(d);
    o[8] = (float)(bits & 0xFFFFFFull);
    o[9] = (float)((bits >> 24) & 0xFFFFFFull);
    o[10] = (float)(bits >> 48);
    o[11] = (float)action;
    const int gm = (int)(ctx.game_id % 101);
    for (int j = 12; j < MZ_O; ++j) o[j] = (float)((j * 37 + k * 11 + gm) % 257) * 0.5f;
}}

__device__ void write_mask(const MzEnvCtx& ctx, int k, MzEnvRow& row) {{
    const int off = (int)(draw(ctx, k, 1) * MZ_A);
    const int p = 1 + (int)(draw(ctx, k, 5) * 4.0);
    const bool one = draw(ctx, k, 6) < 0.25;
    for (int a = 0; a < MZ_A; ++a) row.legal[a] = a == off || (!one && (a + off) % p == 0);
}}

__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {{
    unsigned char* s = static_cast<unsigned char*>(state);
    int count = -1;
#if MZ_SB > 0
    s[0] = (unsigned char)(s[0] + 1);
    count = s[0];
#endif
    const unsigned sum = state_pass(s, -1);
    observe(ctx, row, 0, -1, count, sum);
    if (draw(ctx, 0, 4) >= 0.25) {{
        write_mask(ctx, 0, row);
        *row.to_play = MZ_P > 1 && draw(ctx, 0, 2) < 0.5 ? 1 : 0;
    }}
}}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {{
    unsigned char* s = static_cast<unsigned char*>(state);
    const int k = ctx.move + 1;
    const unsigned sum = state_pass(s, action + ctx.move);
    const int L = 1 + (int)(draw(ctx, 0, 0) * MZ_LMAX);
    const bool done = k >= L;
    *row.reward = (float)(-2.0 + 4.0 * draw(ctx, k, 3));
    *row.done = done;
    if (draw(ctx, k, 4) < 0.2) return;
    int count = -1;
#if MZ_SB > 0
    count = s[0];
#endif
    observe(ctx, row, k, action, count, sum);
    if (done && draw(ctx, k, 7) < 0.5) {{
        for (int a = 0; a < MZ_A; ++a) row.legal[a] = 0;
    }} else {{
        write_mask(ctx, k, row);
    }}
    if (MZ_P > 1 && draw(ctx, k, 2) >= 0.3) *row.to_play = 1 - *row.to_play;
}}
"""


@dataclass(frozen=True)
class Case:
    name: str
    A: int                  # actions
    shape: tuple            # observation_shape (C, H, W)
    stack: int              # stacked_observations
    B: int                  # slots (num_parallel_games)
    state_bytes: int
    P: int                  # players
    max_moves: int

    @property
    def O(self):
        return int(numpy.prod(self.shape))

    @property
    def O_in(self):
        """The search input per slot: (C * (stack + 1) + stack) * H * W (netspec.NetSpec.obs_elems)."""
        C, H, W = self.shape
        return (C * (self.stack + 1) + self.stack) * H * W

    @property
    def lmax(self):
        return self.max_moves + 2

    @property
    def source(self):
        return SOURCE_TEMPLATE.format(A=self.A, O=self.O, P=self.P, SB=self.state_bytes, LMAX=self.lmax, TAG=TAG)


# The edges (selfplay.cu): host_act_kernel<128> up to 128 actions, <256> above; the 256-thread observe / start kernels
# when O_in + A > 4096; the wrapper grid of (B + 127) / 128 CTAs of 128 slots; the state stride of state_bytes rounded
# up to 16.
CASES = {c.name: c for c in [
    Case("single", 1, (1, 1, 12), 0, 1, 0, 1, 4),
    Case("narrow32", 32, (1, 1, 16), 0, 127, 17, 1, 6),
    Case("turns33", 33, (2, 1, 8), 0, 129, 1, 2, 8),
    Case("wide128", 128, (1, 4, 4), 0, 300, 4096, 2, 6),
    Case("wide129", 129, (1, 1, 20), 0, 64, 48, 2, 6),
    Case("wide225", 225, (1, 1, 16), 1, 32, 32, 2, 8),
    Case("wide256", 256, (1, 1, 12), 0, 32, 16, 2, 6),
    Case("row4096", 2, (1, 1, 4094), 0, 16, 32, 1, 6),
    Case("row4097", 2, (1, 1, 1365), 1, 16, 32, 2, 6),
]}


# How the GPU tests play every case: the handle's seed, the first game id and stride (>= B, so a game id gives its slot),
# and the temperature of each call of ``moves_per_call(case)`` moves.
SEED, FIRST_GAME_ID, TEMPERATURES = 11, 7, (1.0, 0.0, 0.5)


def stride_of(case):
    return case.B + 5


def moves_per_call(case):
    return case.max_moves + 2


def finished_games(case, total_moves, seed=SEED, first_game_id=FIRST_GAME_ID, stride=None):
    """The ids of the games the loop finishes in ``total_moves`` moves of every slot.  A game's length depends on its id
    alone (min(L, max_moves)) and a slot starts its next game as soon as one ends, so this needs no search."""
    stride = stride_of(case) if stride is None else stride
    out = []
    for g in range(case.B):
        t, k = 0, 0
        while True:
            gid = first_game_id + g + k * stride
            t += min(planned_length(case, seed, gid), case.max_moves)
            if t > total_moves:
                break
            out.append(gid)
            k += 1
    return out


# ------------------------------------------------------------------------------------------ the rules on the host
class Row:
    """One slot's row as the loop keeps it between calls (selfplay.cu's HostRows)."""

    def __init__(self, case):
        self.obs = numpy.zeros(case.O, numpy.float32)
        self.legal = numpy.ones(case.A, numpy.uint8)
        self.to_play = 0
        self.reward = numpy.float32(0)
        self.done = False


def planned_length(case, seed, gid):
    """The length the rules give game ``gid`` if max_moves does not cut it first."""
    return 1 + int(uniform53(seed, gid, 0, 0, TAG) * case.lmax)


def fp32_operands(seed, gid, k):
    return [numpy.float32(1.0 + uniform53(seed, gid, k, c2, TAG)) for c2 in (8, 9, 10)]


def fp64_operands(seed, gid, k):
    return [1.0 + uniform53(seed, gid, k, c2, TAG) for c2 in (11, 12, 13)]


def fused32(a, b, c):
    """fmaf(a, b, c): with operands in [1, 2) a*b + c is exact in float64, then rounded once."""
    return numpy.float32(numpy.float64(a) * numpy.float64(b) + numpy.float64(c))


def fused64(x, y, z):
    """fma(x, y, z), correctly rounded through exact rationals."""
    return float(Fraction(x) * Fraction(y) + Fraction(z))


class Rules:
    """The case's rules, one slot at a time: ``reset`` / ``step`` update the slot's state bytes and row as the source does
    (the wrappers' defaults included)."""

    def __init__(self, case, seed):
        self.case, self.seed = case, int(seed)
        self._pattern_j = numpy.arange(12, case.O, dtype=numpy.int64)
        self._index = numpy.arange(case.state_bytes, dtype=numpy.int64)

    def draw(self, gid, k, c2):
        return uniform53(self.seed, gid, k, c2, TAG)

    def _checksum(self, state):
        return int((state.astype(numpy.int64) * (self._index + 1)).sum()) & 0xFFFFFFFF

    def _observe(self, row, gid, slot, move, k, action, count, csum):
        o = row.obs
        o[0], o[1], o[2], o[3] = slot, move, gid & 0xFFFFF, gid >> 20
        o[4], o[5], o[6] = count, csum & 0xFFFF, csum >> 16
        a, b, c = fp32_operands(self.seed, gid, k)
        o[7] = a * b + c                                   # float32 multiply, then float32 add
        x, y, z = fp64_operands(self.seed, gid, k)
        bits = struct.unpack("<Q", struct.pack("<d", x * y + z))[0]
        o[8], o[9], o[10] = bits & 0xFFFFFF, (bits >> 24) & 0xFFFFFF, bits >> 48
        o[11] = action
        o[12:] = ((self._pattern_j * 37 + k * 11 + gid % 101) % 257).astype(numpy.float32) * numpy.float32(0.5)

    def _mask(self, row, gid, k):
        A = self.case.A
        off = int(self.draw(gid, k, 1) * A)
        p = 1 + int(self.draw(gid, k, 5) * 4.0)
        one = self.draw(gid, k, 6) < 0.25
        a = numpy.arange(A)
        row.legal[:] = (a == off) | ((not one) & ((a + off) % p == 0))

    def reset(self, state, row, gid, slot):
        row.legal[:] = 1
        row.to_play = 0
        row.reward, row.done = numpy.float32(0), False
        count = -1
        if self.case.state_bytes:
            state[0] = (int(state[0]) + 1) & 255
            count = int(state[0])
        self._observe(row, gid, slot, 0, 0, -1, count, self._checksum(state))
        if self.draw(gid, 0, 4) >= 0.25:
            self._mask(row, gid, 0)
            row.to_play = 1 if self.case.P > 1 and self.draw(gid, 0, 2) < 0.5 else 0

    def step(self, state, row, action, gid, slot, move):
        k = move + 1
        csum = self._checksum(state)
        if self.case.state_bytes > 1:
            state[1:] = ((state[1:].astype(numpy.int64) + action + move + self._index[1:]) & 255).astype(numpy.uint8)
        row.done = k >= planned_length(self.case, self.seed, gid)
        row.reward = numpy.float32(-2.0 + 4.0 * self.draw(gid, k, 3))
        if self.draw(gid, k, 4) < 0.2:
            return
        count = int(state[0]) if self.case.state_bytes else -1
        self._observe(row, gid, slot, move, k, action, count, csum)
        if row.done and self.draw(gid, k, 7) < 0.5:
            row.legal[:] = 0
        else:
            self._mask(row, gid, k)
        if self.case.P > 1 and self.draw(gid, k, 2) >= 0.3:
            row.to_play = 1 - row.to_play


def slot_of(gid, first_game_id, stride):
    """(slot, the slot's game count before this game) of game ``gid``: slot g plays first + g + k * stride."""
    return (gid - first_game_id) % stride, (gid - first_game_id) // stride


def replay(case, seed, first_game_id, stride, games):
    """Replays every finished game of ``games`` ({game id: parse_staged_game dict}) through the rules, a slot's games in
    order from a zero state.  Returns {game id: dict(obs [T + 1, O], reward [T], to_play [T], first_to_play, legal
    [T, A] (the mask each move was chosen under), ending)}; ``ending`` is "first" (done on the first move), "max" (done
    at exactly max_moves), "cut" (max_moves reached in play) or "done".  Raises AssertionError when a record cannot be
    the rules' game: a slot's games not contiguous, an illegal action, or a length the rules do not end at."""
    rules = Rules(case, seed)
    by_slot = {}
    for gid in games:
        slot, k = slot_of(gid, first_game_id, stride)
        assert slot < case.B, (gid, slot)
        by_slot.setdefault(slot, {})[k] = gid
    out = {}
    for slot, ks in by_slot.items():
        assert sorted(ks) == list(range(len(ks))), (slot, sorted(ks))      # no game of the slot missing
        state = numpy.zeros(case.state_bytes, numpy.uint8)
        row = Row(case)
        for k in range(len(ks)):
            gid = ks[k]
            rec = games[gid]
            T = int(rec["length"])
            rules.reset(state, row, gid, slot)
            first_to_play = row.to_play
            obs, reward, to_play, legal = [row.obs.copy()], [], [], []
            for t in range(T):
                assert not row.done, (gid, t, "the rules ended the game before its recorded end")
                a = int(rec["action"][t])
                legal.append(row.legal.copy())
                assert 0 <= a < case.A and row.legal[a], (gid, t, a, "an action illegal under the rules' mask")
                rules.step(state, row, a, gid, slot, t)
                obs.append(row.obs.copy())
                reward.append(row.reward)
                to_play.append(row.to_play)
            L = planned_length(case, seed, gid)
            assert row.done or T == case.max_moves, (gid, T, "the record ends where the rules go on")
            ending = "cut" if not row.done else ("first" if T == 1 else ("max" if T == case.max_moves else "done"))
            assert (L > case.max_moves) == (ending == "cut"), (gid, L, T)
            out[gid] = dict(obs=numpy.stack(obs), reward=numpy.array(reward, numpy.float32),
                            to_play=numpy.array(to_play, numpy.int32), first_to_play=first_to_play,
                            legal=numpy.stack(legal) if legal else numpy.zeros((0, case.A), numpy.uint8), ending=ending)
    return out


# ------------------------------------------------------------------------------------------ plug-in classes
class ContractVector(VectorGame):
    """The rules as the host-stepped route's ``VectorGame``: slot g plays games first + g + k * stride like the device
    loop, so both routes step the same games."""

    def __init__(self, case, num_games, seed, first_game_id, stride):
        self.case, self.num_games = case, int(num_games)
        self.rules = Rules(case, seed)
        self.first, self.stride = int(first_game_id), int(stride)
        self.state = numpy.zeros((self.num_games, case.state_bytes), numpy.uint8)
        self.rows = [Row(case) for _ in range(self.num_games)]
        self.gid = [None] * self.num_games
        self.move = [0] * self.num_games

    def reset(self, which=None):
        for g in range(self.num_games) if which is None else numpy.nonzero(which)[0]:
            self.gid[g] = self.first + g if self.gid[g] is None else self.gid[g] + self.stride
            self.move[g] = 0
            self.rules.reset(self.state[g], self.rows[g], self.gid[g], g)
        return self.observations()

    def observations(self):
        return numpy.stack([r.obs for r in self.rows]).reshape((self.num_games,) + tuple(self.case.shape))

    def step(self, actions, which=None):
        for g in range(self.num_games):
            if which is not None and not which[g]:
                continue
            self.rules.step(self.state[g], self.rows[g], int(actions[g]), self.gid[g], g, self.move[g])
            self.move[g] += 1
        return (self.observations(), numpy.array([r.reward for r in self.rows], numpy.float32),
                numpy.array([r.done for r in self.rows], bool))

    def legal_mask(self):
        return numpy.stack([r.legal for r in self.rows])

    def to_play(self):
        return numpy.array([r.to_play for r in self.rows], numpy.int32)


def make_config(case, **over):
    """A small fully-connected net over the case's shapes; ``over`` sets any other config attribute."""
    class Config(BaseMuZeroConfig):
        _NAME = "user_env_contract_" + case.name
        _OVERRIDES = dict(observation_shape=case.shape, action_space=list(range(case.A)), players=list(range(case.P)),
                          stacked_observations=case.stack, max_moves=case.max_moves, num_simulations=4,
                          num_parallel_games=case.B, rng_mode="philox", support_size=3, encoding_size=4,
                          fc_representation_layers=[], fc_dynamics_layers=[8], fc_reward_layers=[8],
                          fc_value_layers=[8], fc_policy_layers=[8], td_steps=3, PER=True, PER_alpha=1.0)
    cfg = Config()
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def make_game(case, first_game_id, stride, user=True):
    """The case as a plug-in ``Game``: with ``user`` its ``DEVICE_SOURCE`` plays on the device ("device-user-env");
    without, ``vector`` steps the same rules on the host ("device-host-env" with ``config.host_env_device_loop``)."""
    class ContractGame(AbstractGame):
        DEVICE_SOURCE = case.source if user else None
        DEVICE_STATE_BYTES = case.state_bytes

        def __init__(self, seed=None):
            self.seed = seed

        @classmethod
        def vector(cls, num_games, seed=None):
            return ContractVector(case, num_games, seed, first_game_id, stride)

        def step(self, action):
            raise NotImplementedError("the contract games play in batches (vector)")

        def legal_actions(self):
            return list(range(case.A))

        def reset(self):
            raise NotImplementedError("the contract games play in batches (vector)")

        def render(self):
            pass

    return ContractGame


# ------------------------------------------------------------------------------------------ rows the loop cannot play
# The game id's thousands pick the mode, so one source (one compile per handle) serves every case: 0 plays; 1: at move
# 1, slots with slot % 3 == 0 leave their game in play with no legal action and slots with slot % 3 == 1 end it with no
# legal action (allowed); 2: at move 1, slots with slot % 4 == 1 write to_play = num_players; 3: the reset of slots
# with slot % 5 == 2 writes an empty mask.
BAD_ROWS = r"""
__device__ void mz_env_reset(void* state, const MzEnvCtx& ctx, MzEnvRow& row) {
    const int mode = (int)(ctx.game_id / 1000);
    for (int i = 0; i < row.obs_elems; ++i) row.obs[i] = (float)(ctx.slot + i);
    if (mode == 3 && ctx.slot % 5 == 2)
        for (int a = 0; a < row.actions; ++a) row.legal[a] = 0;
}

__device__ void mz_env_step(void* state, int action, const MzEnvCtx& ctx, MzEnvRow& row) {
    const int mode = (int)(ctx.game_id / 1000);
    *row.reward = 1.0f;
    row.obs[0] = (float)ctx.move;
    if (ctx.move != 1) return;
    if (mode == 1 && ctx.slot % 3 < 2) {
        for (int a = 0; a < row.actions; ++a) row.legal[a] = 0;
        *row.done = ctx.slot % 3 == 1;
    }
    if (mode == 2 && ctx.slot % 4 == 1) *row.to_play = row.num_players;
}
"""


def bad_rows_expected(mode, B, A, P):
    """The rows mz_env_check counts for BAD_ROWS's ``mode`` over B slots: the reset's (mode 3) or move 1's (modes 1, 2) -
    a to_play outside [0, P), or a row still in play (reset, or not done) without a legal action."""
    bad = 0
    for g in range(B):
        legal, to_play, done = numpy.ones(A, bool), 0, False
        if mode == 3 and g % 5 == 2:
            legal[:] = False
        if mode == 1 and g % 3 < 2:
            legal[:], done = False, g % 3 == 1
        if mode == 2 and g % 4 == 1:
            to_play = P
        bad += (not 0 <= to_play < P) or (not done and not legal.any())
    return bad


# ------------------------------------------------------------------------------------------ the edges
def edges(case):
    """The launch and layout edges the case reaches, by selfplay.cu's formulas."""
    return dict(act_kernel=128 if case.A <= 128 else 256,
                slot_threads=256 if case.O_in + case.A > 4096 else 32,
                wrapper_ctas=(case.B + 127) // 128, partial_cta=case.B % 128 != 0,
                state_stride=(case.state_bytes + 15) & ~15)


def coverage(case, gids, seed=SEED):
    """What the finished games ``gids`` reach, from their draws alone (no move depends on the actions): their endings,
    terminal rows without a legal action, moves with one legal action (A > 1), steps that write only reward and done,
    resets that keep the default mask and to_play, games player 1 opens, moves after which the same player moves again."""
    rules = Rules(case, seed)
    out = dict(first=0, max=0, cut=0, done=0, empty_terminal=0, one_legal=0, partial=0, default_reset=0, opens_1=0,
               same_player=0)
    for gid in gids:
        L = planned_length(case, seed, gid)
        T = min(L, case.max_moves)
        out["cut" if L > case.max_moves else "first" if T == 1 else "max" if T == case.max_moves else "done"] += 1
        written = rules.draw(gid, 0, 4) >= 0.25
        out["default_reset"] += not written
        out["opens_1"] += written and case.P > 1 and rules.draw(gid, 0, 2) < 0.5
        out["one_legal"] += written and case.A > 1 and rules.draw(gid, 0, 6) < 0.25
        for k in range(1, T + 1):
            partial = rules.draw(gid, k, 4) < 0.2
            out["partial"] += partial
            if case.P > 1 and k < T:
                out["same_player"] += partial or rules.draw(gid, k, 2) < 0.3
            if partial:
                continue
            if k == L:
                out["empty_terminal"] += rules.draw(gid, k, 7) < 0.5
            elif k < T:
                out["one_legal"] += case.A > 1 and rules.draw(gid, k, 6) < 0.25
    return out


def contraction_differs(seed, gids, moves):
    """(fp32, fp64): whether some observation's ``a * b + c`` over the draws of games ``gids`` at k = 0 .. moves
    differs between the unfused (the source's) and fused roundings."""
    d32 = d64 = False
    for gid in gids:
        for k in range(moves + 1):
            a, b, c = fp32_operands(seed, gid, k)
            d32 |= bool(a * b + c != fused32(a, b, c))
            x, y, z = fp64_operands(seed, gid, k)
            d64 |= x * y + z != fused64(x, y, z)
            if d32 and d64:
                return True, True
    return d32, d64


def _check_fraction_fma():
    # the exact-rational fma must round like IEEE fma: a classic case where the fused result keeps the product's tail
    x = 1.0 + 2.0 ** -30
    assert fused64(x, x, -1.0) == 2.0 ** -29 + 2.0 ** -60 and x * x - 1.0 == 2.0 ** -29
    assert math.isclose(fused64(1.5, 1.25, 1.0), 2.875)


_check_fraction_fma()
