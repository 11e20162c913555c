"""Struct-of-arrays board games (numpy) shared by the TicTacToe and Connect4 plug-ins.

Rules and observation planes follow the reference environments
(``games/tictactoe.py:243-306``, ``games/connect4.py:220-305``): three planes
``[stones of player +1, stones of player -1, constant plane = side to move (+1/-1)]``,
player +1 moves first and is ``to_play() == 0``; the mover gets reward 1 on completing a
line, the game also ends when the board is full.  Winning lines are precomputed as index
tables, so a whole batch is checked with one gather.
"""
import copy

import numpy

from .abstract_game import VectorGame


def _lines(h, w, k):
    out = []
    for r in range(h):
        for c in range(w):
            for dr, dc in ((0, 1), (1, 0), (1, 1), (-1, 1)):
                cells = [(r + i * dr, c + i * dc) for i in range(k)]
                if all(0 <= y < h and 0 <= x < w for y, x in cells):
                    out.append([y * w + x for y, x in cells])
    return numpy.array(out, dtype=numpy.int64)


class BoardVector(VectorGame):
    H = W = K = 0
    GRAVITY = False            # Connect4: a move names a column and the stone drops
    OBS_DTYPE = numpy.float64
    REWARD_SCALE = 1
    REWARD_WHEN_FULL = False   # games/gomoku.py:243-247 pays the mover whenever the game ends, a full board included

    def __init__(self, num_games, seed=None):
        self.num_games = int(num_games)
        self.lines = _lines(self.H, self.W, self.K)
        self.board = numpy.zeros((self.num_games, self.H * self.W), dtype=numpy.int32)
        self.player = numpy.ones(self.num_games, dtype=numpy.int32)

    # ----------------------------------------------------------------------------
    def reset(self, which=None):
        if which is None:
            self.board[:] = 0
            self.player[:] = 1
        else:
            self.board[which] = 0
            self.player[which] = 1
        return self.observations()

    def observations(self):
        b = self.board.reshape(self.num_games, self.H, self.W)
        obs = numpy.empty((self.num_games, 3, self.H, self.W), dtype=self.OBS_DTYPE)
        obs[:, 0] = b == 1
        obs[:, 1] = b == -1
        obs[:, 2] = self.player[:, None, None]
        return obs

    def to_play(self):
        return numpy.where(self.player == 1, 0, 1).astype(numpy.int32)

    def legal_mask(self):
        if self.GRAVITY:
            top = self.board.reshape(self.num_games, self.H, self.W)[:, self.H - 1, :]
            return (top == 0).astype(numpy.uint8)
        return (self.board == 0).astype(numpy.uint8)

    def step(self, actions, which=None):
        """Steps every game, or the games of the bool mask ``which`` (the others keep their state and report reward 0,
        not done)."""
        if which is not None:
            g = numpy.nonzero(which)[0]
            sub = copy.copy(self)
            sub.num_games, sub.board, sub.player = len(g), self.board[g], self.player[g]
            r, d = sub._step_all(numpy.asarray(actions, dtype=numpy.int64)[g])
            self.board[g], self.player[g] = sub.board, sub.player
            reward, done = numpy.zeros(self.num_games, r.dtype), numpy.zeros(self.num_games, bool)
            reward[g], done[g] = r, d
            return self.observations(), reward, done
        reward, done = self._step_all(actions)
        return self.observations(), reward, done

    def _step_all(self, actions):
        actions = numpy.asarray(actions, dtype=numpy.int64)
        g = numpy.arange(self.num_games)
        if self.GRAVITY:
            cols = self.board.reshape(self.num_games, self.H, self.W)[g, :, actions]   # [n, H]
            free = cols == 0
            row = numpy.argmax(free, axis=1)                # lowest empty row
            ok = free.any(axis=1)                           # a full column leaves the board unchanged
            cell = row * self.W + actions
            self.board[g[ok], cell[ok]] = self.player[ok]
        else:
            self.board[g, actions] = self.player
        mine = self.board == self.player[:, None]
        won = mine[:, self.lines].all(axis=2).any(axis=1)
        full = ~(self.legal_mask().any(axis=1))
        reward = numpy.where(won | full if self.REWARD_WHEN_FULL else won, 1, 0) * self.REWARD_SCALE
        self.player = -self.player
        return reward, won | full

    @staticmethod
    def expert_windows(board):
        """The windows of the game's hard-coded opponent for ``_threat_scan``, in the reference's scan order."""
        raise NotImplementedError("this game has no expert opponent (the reference's Game has no expert_agent)")

    def expert_actions(self, defaults, which):
        """``BoardGame.expert_agent`` of the games of the bool mask ``which``, each with the random fallback
        ``defaults[g]`` in place of its ``numpy.random.choice`` draw; -1 for the others."""
        out = numpy.full(self.num_games, -1, numpy.int32)
        boards = self.board.reshape(self.num_games, self.H, self.W)
        for g in numpy.nonzero(which)[0]:
            out[g] = _threat_scan(boards[g], int(self.player[g]), self.expert_windows(boards[g]), int(defaults[g]))
        return out


def _threat_scan(board, player, windows, default):
    """Shared core of the reference's hard-coded opponents (``games/tictactoe.py:310-349``,
    ``games/connect4.py:307-348``): walk ``windows`` - tuples ``(cells, need, playable)`` - in the reference's
    scan order; a window whose stones sum to +-``need`` has exactly one empty cell: that cell's action becomes the
    candidate if ``playable(cell)`` holds, and is returned at once when the window belongs to the side to move (a win);
    otherwise (a block) the scan continues and a later window may overwrite the candidate."""
    action = default
    for cells, need, playable, fixed_action in windows:
        vals = [int(board[y][x]) for y, x in cells]
        total = sum(vals)
        if abs(total) != need:
            continue
        if fixed_action is not None:                  # Connect4's vertical check names the column without looking for the gap
            action = fixed_action
        else:
            y, x = cells[vals.index(0)]
            if not playable(y, x):
                continue
            action = playable.action(y, x)
        if player * total > 0:
            return action
    return action


class BoardGame:
    """Single-game facade over a one-game ``BoardVector`` with reference return types."""
    VECTOR = BoardVector

    def __init__(self, seed=None):
        self.env = self.VECTOR(1, seed)

    @classmethod
    def vector(cls, num_games, seed=None):
        return cls.VECTOR(num_games, seed)

    def step(self, action):
        obs, reward, done = self.env.step(numpy.array([action]))
        return obs[0], int(reward[0]), bool(done[0])

    def to_play(self):
        return int(self.env.to_play()[0])

    def legal_actions(self):
        return [int(a) for a in numpy.nonzero(self.env.legal_mask()[0])[0]]

    @classmethod
    def legal_masks(cls, observations):
        """The legal mask of each raw frame [n, 3, H, W] (Reanalyse's hook), read from the stone planes: the empty
        cells, or with gravity the columns whose top cell ``board[H - 1][c]`` is empty.  The side comes from the shape."""
        obs = numpy.asarray(observations)
        empty = (obs[:, 0] == 0) & (obs[:, 1] == 0)
        if cls.VECTOR.GRAVITY:
            return empty[:, -1, :].astype(numpy.uint8)
        return empty.reshape(len(obs), obs.shape[2] * obs.shape[3]).astype(numpy.uint8)

    def reset(self):
        return self.env.reset()[0]

    def render(self):
        print(self.env.board[0].reshape(self.env.H, self.env.W)[::-1])

    def close(self):
        pass

    def expert_agent(self):
        """Hard-coded opponent of the evaluation worker (``self_play.py:211-212``).  Like the reference it first
        draws a uniformly random legal action from the global ``numpy.random`` stream (consumed even when a threat is
        found), then scans for a winning move / a move that blocks the opponent."""
        env = self.env
        H, W = env.H, env.W
        board = env.board[0].reshape(H, W)
        player = int(env.player[0])
        default = numpy.random.choice(self.legal_actions())
        return _threat_scan(board, player, self._expert_windows(board), default)

    def _expert_windows(self, board):
        return self.VECTOR.expert_windows(board)
