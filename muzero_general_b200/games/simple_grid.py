"""Simple Grid plug-in (config values and rules of the reference's ``games/simple_grid.py``): walk from (0, 0) to the
corner (2, 2) of a 3 x 3 grid, down or right; the observation is the one-hot position."""
import numpy

from ._config import BaseMuZeroConfig
from .abstract_game import AbstractGame, VectorGame


class MuZeroConfig(BaseMuZeroConfig):
    _NAME = "simple_grid"
    _OVERRIDES = dict(
        observation_shape=(1, 1, 9), max_moves=6, num_simulations=10, discount=0.978,
        encoding_size=5, fc_representation_layers=[16],
        training_steps=30000, batch_size=32, lr_init=0.0064, lr_decay_rate=1, lr_decay_steps=1000,
        replay_buffer_size=5000, num_unroll_steps=7, td_steps=7, self_play_delay=0.2, ratio=None,
    )
    _TEMPERATURE_SCHEDULE = ((None, 1),)


class SimpleGridVector(VectorGame):
    """``num_games`` grids (``GridEnv``, games/simple_grid.py:192-229): action 0 adds 1 to the row, 1 to the column; a
    move off the edge changes nothing; reaching (2, 2) pays ``REWARD_SCALE`` (``Game.step``'s x10) and ends the game."""
    SIZE = 3
    OBS_DTYPE = numpy.float64
    REWARD_SCALE = 10

    def __init__(self, num_games, seed=None):
        self.num_games = int(num_games)
        self.pos = numpy.zeros((self.num_games, 2), dtype=numpy.int64)

    def reset(self, which=None):
        if which is None:
            self.pos[:] = 0
        else:
            self.pos[which] = 0
        return self.observations()

    def observations(self):
        obs = numpy.zeros((self.num_games, 1, 1, self.SIZE * self.SIZE), dtype=self.OBS_DTYPE)
        obs[numpy.arange(self.num_games), 0, 0, self.pos[:, 0] * self.SIZE + self.pos[:, 1]] = 1
        return obs

    def legal_mask(self):
        return numpy.ones((self.num_games, 2), dtype=numpy.uint8)      # Game.legal_actions, not GridEnv's

    def step(self, actions):
        a = numpy.asarray(actions, dtype=numpy.int64)
        g = numpy.arange(self.num_games)
        self.pos[g, a] = numpy.minimum(self.pos[g, a] + 1, self.SIZE - 1)
        done = (self.pos == self.SIZE - 1).all(axis=1)
        return self.observations(), done.astype(numpy.int64) * self.REWARD_SCALE, done


class Game(AbstractGame):
    DEVICE_ENV = "simple_grid"      # csrc/selfplay.cu restates these rules on the device
    VECTOR = SimpleGridVector

    def __init__(self, seed=None):
        self.env = SimpleGridVector(1, seed)

    @classmethod
    def vector(cls, num_games, seed=None):
        return SimpleGridVector(num_games, seed)

    def step(self, action):
        obs, reward, done = self.env.step(numpy.array([action]))
        return obs[0], int(reward[0]), bool(done[0])

    def legal_actions(self):
        return list(range(2))

    @staticmethod
    def legal_masks(observations):
        """The legal mask of each raw frame [n, *observation_shape] (Reanalyse's hook): every action, as legal_actions."""
        return numpy.ones((len(observations), 2), numpy.uint8)

    def reset(self):
        return self.env.reset()[0]

    def render(self):
        im = numpy.full((3, 3), "-")
        im[2, 2] = "1"
        im[self.env.pos[0, 0], self.env.pos[0, 1]] = "x"
        print(im)

    def action_to_string(self, action_number):
        return f"{action_number}. " + ("Down", "Right")[action_number]
