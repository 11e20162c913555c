"""Gridworld plug-in (config values of the reference's ``games/gridworld.py``) without gym_minigrid.

The reference wraps ``gym.make("MiniGrid-Empty-Random-6x6-v0")`` behind ``gym_minigrid.wrappers.ImgObsWrapper``.
gym_minigrid is a third-party package that is neither vendored in the reference nor in its ``requirements.lock``, so
the rules of gym_minigrid 1.0.x (``MiniGridEnv``, ``EmptyEnv(size=6, agent_start_pos=None)``, ``ImgObsWrapper``) are
restated here as a struct-of-arrays numpy environment.  PARITY UNPINNED against gym_minigrid (absent), as with
CartPole and gym.  ``csrc/selfplay.cu`` (``MZ_ENV_GRIDWORLD``) plays the same rules on the device.

The rules:

* Grid: 6 x 6, cells ``(x, y)``; every cell with x or y in {0, 5} is a wall, the goal is at (4, 4), the rest is empty.
* Reset: the agent takes a uniformly random free cell (one of the 15 cells with 1 <= x, y <= 4 other than the goal)
  and a uniformly random direction in 0..3 (0 = +x, 1 = +y, 2 = -x, 3 = -y); ``step_count = 0``.
* Step: ``step_count += 1``; action 0 turns left (``dir = (dir + 3) % 4``), 1 turns right (``dir = (dir + 1) % 4``),
  2 moves to the cell ahead unless it is a wall.  Entering the goal ends the game with reward
  ``1 - 0.9 * (step_count / 144)`` (fp64; ``max_steps = 4 * 6 * 6``); otherwise the reward is 0, and the game also
  ends when ``step_count >= 144``.  The legal actions are always [0, 1, 2] (the reference's ``Game.legal_actions``).
* Observation (``ImgObsWrapper``'s ``obs["image"]``): uint8 ``(7, 7, 3)`` indexed ``[x'][y'][channel]``.  The 7 x 7
  window with top-left corner (ax, ay - 3), (ax - 3, ay), (ax - 6, ay - 3) or (ax - 3, ay - 6) for dir 0, 1, 2 or 3
  is sliced from the grid (cells outside it read as walls), rotated left dir + 1 times (one rotation:
  ``new[j][6 - i] = old[i][j]``), the agent's own cell (3, 6) is set to empty, and every cell is encoded as empty
  (1, 0, 0), wall (2, 5, 0) or goal (8, 1, 0).  The room sees through walls, so no cell is unseen.
* Network input: ``torch.tensor(observation).float()``, the 147 values in ``[x'][y'][c]`` order.

The placement source is pluggable: by default ``numpy.random.RandomState(seed)`` in MiniGrid's draw order
(``randint(0, 6)`` for x, then y, again on a taken cell, then ``randint(0, 4)`` for the direction), and the same rules
replay any other source, the device's Philox placement included (``oracle/gridworld.py``).
"""
import numpy

from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame, VectorGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "gridworld"
    _OVERRIDES = dict(
        observation_shape=(7, 7, 3), action_space=list(range(3)), num_workers=4, max_moves=15, num_simulations=20,
        training_steps=30000, lr_init=0.005, lr_decay_rate=1, replay_buffer_size=5000, td_steps=20, PER=False,
        use_last_model_value=False, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((0.5, 1.0), (0.75, 0.5), (None, 0.25))


SIZE = 6
GOAL = (4, 4)
MAX_STEPS = 4 * SIZE * SIZE
VIEW = 7
EMPTY, WALL, GOAL_CELL = 0, 1, 2
ENCODING = numpy.array([[1, 0, 0], [2, 5, 0], [8, 1, 0]], dtype=numpy.uint8)     # empty, wall (grey), goal (green)
DIRECTIONS = numpy.array([[1, 0], [0, 1], [-1, 0], [0, -1]], dtype=numpy.int64)
_VIEW_TOP = ((0, -3), (-3, 0), (-6, -3), (-3, -6))      # window corner - agent, per direction


def _rotate_left(grid):
    """``Grid.rotate_left``: new[j][VIEW - 1 - i] = old[i][j]."""
    new = [[None] * VIEW for _ in range(VIEW)]
    for i in range(VIEW):
        for j in range(VIEW):
            new[j][VIEW - 1 - i] = grid[i][j]
    return new


def _view_offsets():
    """[dir][x'][y'] -> the grid offset from the agent of view cell (x', y'): the window of the rules, rotated."""
    out = numpy.zeros((4, VIEW, VIEW, 2), dtype=numpy.int64)
    for d, (tx, ty) in enumerate(_VIEW_TOP):
        window = [[(tx + i, ty + j) for j in range(VIEW)] for i in range(VIEW)]
        for _ in range(d + 1):
            window = _rotate_left(window)
        out[d] = window
    return out


VIEW_OFFSETS = _view_offsets()
_PAD = VIEW - 1                  # every view cell of an agent on the grid lies within PAD cells of it


def _cells():
    """The grid's objects, padded by _PAD wall cells on every side: cells[x + _PAD][y + _PAD]."""
    n = SIZE + 2 * _PAD
    cells = numpy.full((n, n), WALL, dtype=numpy.int64)
    cells[_PAD + 1:_PAD + SIZE - 1, _PAD + 1:_PAD + SIZE - 1] = EMPTY
    cells[_PAD + GOAL[0], _PAD + GOAL[1]] = GOAL_CELL
    return cells


CELLS = _cells()


def numpy_placement(seed):
    """MiniGrid's ``place_agent`` on ``RandomState(seed)``: x = ``randint(0, 6)``, then y, drawn again while the cell
    is a wall or the goal, then the direction ``randint(0, 4)``."""
    rs = numpy.random.RandomState(seed)

    def place():
        while True:
            x, y = int(rs.randint(0, SIZE)), int(rs.randint(0, SIZE))
            if CELLS[x + _PAD, y + _PAD] == EMPTY:
                return x, y, int(rs.randint(0, 4))
    return place


class GridworldVector(VectorGame):
    """``num_games`` rooms of the rules above.  ``places[g]`` is game g's placement source, a callable returning the
    next game's (x, y, dir); by default ``numpy_placement(seed + g)``."""
    OBS_DTYPE = numpy.uint8
    REWARD_TYPE = float

    def __init__(self, num_games, seed=None, places=None):
        self.num_games = int(num_games)
        if places is None:
            places = [numpy_placement(None if seed is None else seed + g) for g in range(self.num_games)]
        self.places = list(places)
        self.x = numpy.zeros(self.num_games, dtype=numpy.int64)
        self.y = numpy.zeros(self.num_games, dtype=numpy.int64)
        self.dir = numpy.zeros(self.num_games, dtype=numpy.int64)
        self.step_count = numpy.zeros(self.num_games, dtype=numpy.int64)

    def reset(self, which=None):
        idx = range(self.num_games) if which is None else numpy.arange(self.num_games)[numpy.asarray(which)]
        for g in idx:
            self.x[g], self.y[g], self.dir[g] = self.places[g]()
            self.step_count[g] = 0
        return self.observations()

    def observations(self):
        off = VIEW_OFFSETS[self.dir]                                               # [n, 7, 7, 2]
        obj = CELLS[self.x[:, None, None] + off[..., 0] + _PAD, self.y[:, None, None] + off[..., 1] + _PAD]
        obj[:, VIEW // 2, VIEW - 1] = EMPTY                                        # the agent's own cell
        return ENCODING[obj]

    def legal_mask(self):
        return numpy.ones((self.num_games, 3), dtype=numpy.uint8)

    def step(self, actions):
        a = numpy.asarray(actions, dtype=numpy.int64)
        self.step_count += 1
        ahead = DIRECTIONS[self.dir]
        fx, fy = self.x + ahead[:, 0], self.y + ahead[:, 1]
        obj = CELLS[fx + _PAD, fy + _PAD]
        move = (a == 2) & (obj != WALL)
        self.x, self.y = numpy.where(move, fx, self.x), numpy.where(move, fy, self.y)
        self.dir = numpy.where(a == 0, (self.dir + 3) % 4, numpy.where(a == 1, (self.dir + 1) % 4, self.dir))
        goal = move & (obj == GOAL_CELL)
        reward = numpy.where(goal, 1 - 0.9 * (self.step_count / MAX_STEPS), 0.0)
        done = goal | (self.step_count >= MAX_STEPS)
        return self.observations(), reward, done


class Game(AbstractGame):
    DEVICE_ENV = "gridworld"        # csrc/selfplay.cu restates these rules on the device
    VECTOR = GridworldVector

    def __init__(self, seed=None):
        self.env = GridworldVector(1, seed)

    @classmethod
    def vector(cls, num_games, seed=None):
        return GridworldVector(num_games, seed)

    def step(self, action):
        obs, reward, done = self.env.step(numpy.array([action]))
        return obs[0], float(reward[0]), bool(done[0])

    def legal_actions(self):
        return list(range(3))

    @staticmethod
    def legal_masks(observations):
        """The legal mask of each raw frame [n, *observation_shape] (Reanalyse's hook): every action, as legal_actions."""
        return numpy.ones((len(observations), 3), numpy.uint8)

    def reset(self):
        return self.env.reset()[0]

    def render(self):
        im = numpy.full((SIZE, SIZE), " ")
        im[CELLS[_PAD:_PAD + SIZE, _PAD:_PAD + SIZE] == WALL] = "#"
        im[GOAL] = "G"
        im[self.env.x[0], self.env.y[0]] = ">v<^"[self.env.dir[0]]
        print("\n".join("".join(im[:, y]) for y in range(SIZE)))

    def action_to_string(self, action_number):
        actions = {
            0: "Turn left",
            1: "Turn right",
            2: "Move forward",
            3: "Pick up an object",
            4: "Drop the object being carried",
            5: "Toggle (open doors, interact with objects)",
        }
        return f"{action_number}. {actions[action_number]}"
